"""ctypes binding of include/lc_b200.h.  Host arrays are numpy; device pointers are plain ints
(e.g. ``torch.Tensor.data_ptr()``) -- torch is only plumbing for HBM allocations and streams."""
import ctypes as C
import os

import numpy as np

from . import _build

LC_OK, LC_ERR_INVALID_ARG, LC_ERR_CUDA, LC_ERR_REGEX_INVALID, LC_ERR_REGEX_UNSUPPORTED, LC_ERR_CAPACITY, \
    LC_ERR_TOO_LARGE = range(7)
LC_ML_IS_LAST, LC_ML_MATCHED = 1, 2

_LIB = None


class LcError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("lc_b200 error %d: %s" % (code, msg))
        self.code = code


def lib():
    """Loads libloongcollector_b200.so (building it in-tree if sources are newer). Raises if unavailable."""
    global _LIB
    if _LIB is not None:
        return _LIB
    so = _build.SO
    if _build.needs_build():
        if os.path.exists("/usr/local/cuda/bin/nvcc") or os.environ.get("NVCC"):
            _build.build()
        elif not os.path.exists(so):
            raise ImportError("libloongcollector_b200.so is missing and nvcc is not available; "
                              "run `python -m loongcollector_b200._build` (there is no CPU fallback)")
    L = C.CDLL(so)
    vp, u64, u32, u8, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint8, C.c_int
    L.lc_version.restype = C.c_char_p
    L.lc_last_error.restype = C.c_char_p
    L.lc_device_count.restype = i32
    L.lc_engine_create.argtypes = [i32, C.POINTER(vp)]
    L.lc_engine_destroy.argtypes = [vp]
    L.lc_engine_sync.argtypes = [vp]
    L.lc_engine_stream.restype = vp
    L.lc_engine_stream.argtypes = [vp]
    L.lc_engine_launch_count.restype = u64
    L.lc_engine_launch_count.argtypes = [vp]
    L.lc_host_alloc.restype = vp
    L.lc_host_alloc.argtypes = [C.c_size_t]
    L.lc_host_free.argtypes = [vp]
    L.lc_regex_compile.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(vp)]
    L.lc_regex_free.argtypes = [vp]
    L.lc_regex_error.restype = C.c_char_p
    L.lc_regex_error.argtypes = [vp]
    L.lc_regex_ngroups.restype = u32
    L.lc_regex_ngroups.argtypes = [vp]
    L.lc_regex_info.argtypes = [vp, vp]
    split_args = [vp, vp, u64, u8, vp, vp, u64, C.POINTER(u64)]
    L.lc_split_lines.argtypes = split_args
    L.lc_split_lines_dev.argtypes = split_args
    parse_args = [vp, vp, vp, u64, vp, vp, u64, u32, vp, vp, vp]
    L.lc_regex_parse.argtypes = parse_args
    L.lc_regex_parse_dev.argtypes = parse_args
    L.lc_engine_set_stream.argtypes = [vp, vp]
    L.lc_regex_parse_strided_dev.argtypes = [vp, vp, vp, u64, vp, vp, u32, u64, u32, vp, vp, vp]
    multi_args = [vp, vp, u32, vp, vp, u64, vp, vp, u64, vp, vp, vp, u32, vp, vp]
    L.lc_regex_parse_multi.argtypes = multi_args
    L.lc_regex_parse_multi_dev.argtypes = multi_args
    rl_args = [vp, vp, u64, vp, vp, i32, C.POINTER(u64), C.POINTER(C.c_int32)]
    L.lc_remove_last_incomplete_log.argtypes = rl_args
    L.lc_remove_last_incomplete_log_dev.argtypes = rl_args
    L.lc_sls_serialize_parsed_dev.argtypes = [vp, vp, u64, vp, vp, vp, vp, vp, u32, u64, vp, vp, u32, C.c_char_p, u32, vp,
                                              vp, vp, u64, C.POINTER(u64)]
    L.lc_regex_prefix_match.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp]
    L.lc_regex_match.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp]
    L.lc_regex_match_dev.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp]
    ml_args = [vp, vp, u64, vp, vp, vp, i32, vp, vp, vp, u64, C.POINTER(u64), vp]
    L.lc_multiline_split.argtypes = ml_args
    L.lc_multiline_split_dev.argtypes = ml_args
    dl_args = [vp, vp, u64, vp, vp, u64, vp, u32, u8, u32, i32, i32, u32, vp, vp, vp, vp, vp]
    L.lc_delim_parse.argtypes = dl_args
    L.lc_delim_parse_dev.argtypes = dl_args
    L.lc_delim_parse_tap_dev.argtypes = dl_args + [u32, vp, vp]
    L.lc_delim_regex_chain.argtypes = dl_args + [u32, vp, u32, vp, vp, vp]
    L.lc_sls_serialize_logs.argtypes = [vp, vp, u64, u64, vp, vp, vp, vp, vp, vp, vp, vp, u64, C.POINTER(u64)]
    sls_cfg = [vp, vp, u32, C.c_char_p, u32, C.c_char_p, u32, i32, i32, i32]  # keys .. copy_raw
    L.lc_sls_serialize_delim_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp, u32, vp, u32, u8, i32,
                                             i32] + sls_cfg + [vp, vp, vp, u64, C.POINTER(u64)]
    L.lc_delim_parse_sls.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, u32, u8, i32, i32, i32, u32] + sls_cfg + \
        [vp, u64, C.POINTER(u64), vp]
    L.lc_sls_serialize_regex_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, u32] + sls_cfg + \
        [i32, vp, vp, vp, u64, C.POINTER(u64), vp]
    L.lc_regex_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp, vp] + sls_cfg + [i32, vp, u64, C.POINTER(u64), vp]
    span_keys = [C.c_char_p, u32, C.c_char_p, u32, u64, u32, u32]  # key .. time_ns
    L.lc_sls_serialize_spans_dev.argtypes = [vp, vp, u64, vp, vp, u64] + span_keys + [vp, u64, C.POINTER(u64)]
    L.lc_split_sls.argtypes = [vp, vp, u64, u8] + span_keys + [vp, u64, C.POINTER(u64), C.POINTER(u64)]
    L.lc_multiline_split_sls.argtypes = [vp, vp, u64, vp, vp, vp, i32] + span_keys + [vp, u64, C.POINTER(u64),
                                                                                         C.POINTER(u64), vp]
    L.lc_lz4_compress_dev.argtypes = [vp, vp, u64, vp, vp, vp, u64, vp, vp, C.POINTER(u64)]
    L.lc_lz4_compress.argtypes = [vp, u64, vp, vp, vp, u64, vp, vp, C.POINTER(u64)]
    L.lc_zstd_compress_dev.argtypes = [vp, vp, u64, vp, vp, vp, u64, vp, vp, C.POINTER(u64)]
    L.lc_zstd_compress.argtypes = [vp, u64, vp, vp, vp, u64, vp, vp, C.POINTER(u64)]
    L.lc_timestamp_compile.argtypes = [C.c_char_p, C.c_size_t, i32, i32, C.POINTER(vp)]
    L.lc_timestamp_free.argtypes = [vp]
    ts_tail = [vp, u64, C.c_int64, i32, vp, vp, vp, vp]  # grp .. counters
    L.lc_timestamp_parse.argtypes = [vp, vp, vp, u64, vp, vp, u64] + ts_tail
    L.lc_timestamp_parse_dev.argtypes = [vp, vp, vp, u64, vp, vp, u64] + ts_tail
    L.lc_timestamp_parse_capture_dev.argtypes = [vp, vp, vp, u64, vp, vp, vp, u32, u32, u64] + ts_tail
    L.lc_apsara_compile.argtypes = [C.c_char_p, C.c_size_t, i32, C.POINTER(vp)]
    L.lc_apsara_free.argtypes = [vp]
    ap_args = [vp, vp, vp, u64, vp, vp, u64, vp, u64, C.c_int64, i32, vp, vp, vp, vp, vp, vp, u64, C.POINTER(u64), vp]
    L.lc_apsara_parse.argtypes = ap_args
    L.lc_apsara_parse_dev.argtypes = ap_args
    L.lc_json_compile.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(vp)]
    L.lc_json_free.argtypes = [vp]
    js_args = [vp, vp, vp, u64, vp, vp, u64, vp, vp, vp, u64, C.POINTER(u64), vp, u64, C.POINTER(u64), vp]
    L.lc_json_parse.argtypes = js_args
    L.lc_json_parse_dev.argtypes = js_args
    L.lc_delim_parse_sls_lz4.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, u32, u8, i32, i32, i32, u32] + \
        sls_cfg + [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_regex_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp, vp] + sls_cfg + \
        [i32, vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    chain_cfg = [vp, u32, u8, i32, i32] + sls_cfg + sls_cfg + [i32]  # sep .. copy_raw, rkeys .. rcopy_raw, whole_line
    dtab = [vp, vp, u64, vp, vp, vp, vp, vp, u32]  # d_ev_off .. max_fields
    L.lc_delim_regex_tap_dev.argtypes = [vp, vp, u64, u64] + dtab + chain_cfg + [vp, vp, C.POINTER(u64)]
    L.lc_sls_serialize_delim_regex_dev.argtypes = [vp, vp, u64] + dtab + chain_cfg + \
        [vp, vp, vp, vp, vp, u32, vp, vp, vp, u64, C.POINTER(u64), vp]
    L.lc_delim_regex_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp, vp, i32, u32] + chain_cfg + \
        [vp, u64, C.POINTER(u64), vp]
    L.lc_delim_regex_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp, vp, i32, u32] + chain_cfg + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    sr_tail = [C.c_char_p, u32, u64, u32, u32]  # offset_key .. time_ns of the split -> regex chain
    sj_cfg = [C.c_char_p, u32, i32, i32, i32] + sr_tail  # renamed_key .. time_ns of the split -> JSON chain
    L.lc_sls_serialize_split_json_dev.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp, vp, vp, vp] + sj_cfg + \
        [vp, u64, C.POINTER(u64), vp]
    L.lc_split_json_parse_sls.argtypes = [vp, vp, vp, u64, u8] + sj_cfg + [vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_json_parse_sls_lz4.argtypes = [vp, vp, vp, u64, u8] + sj_cfg + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_json_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sj_cfg + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_json_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sj_cfg + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    # the split -> JSON -> timestamp chain: the split -> JSON arguments with the timestamp stage behind time_ns
    sjt_ts = [C.c_char_p, u32, vp, C.c_int64, i32, i32]  # tkey, tkey_len, ts, now, discard_interval, enable_ns
    L.lc_split_json_timestamp_tap_dev.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, C.c_char_p, u32, i32,
                                                  i32, i32, C.c_char_p, u32, C.c_char_p, u32, vp, u64, vp, vp]
    L.lc_sls_serialize_split_json_timestamp_dev.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp, vp, vp, vp] + sj_cfg + \
        [vp, vp, vp, i32, vp, u64, C.POINTER(u64), vp]
    L.lc_split_json_timestamp_parse_sls.argtypes = [vp, vp, vp, u64, u8] + sj_cfg + sjt_ts + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_json_timestamp_parse_sls_lz4.argtypes = [vp, vp, vp, u64, u8] + sj_cfg + sjt_ts + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_json_timestamp_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sj_cfg + sjt_ts + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_json_timestamp_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sj_cfg + \
        sjt_ts + [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    sa_cfg = [C.c_char_p, u32, i32, i32, i32] + sr_tail + [i32]  # renamed_key .. enable_ns of the split -> Apsara chain
    sa_now = [C.c_int64, i32]  # now, discard_interval
    L.lc_sls_serialize_split_apsara_dev.argtypes = [vp, vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp, vp] + sa_cfg + \
        [vp, u64, C.POINTER(u64), vp]
    L.lc_split_apsara_parse_sls.argtypes = [vp, vp, vp, u64, u8] + sa_cfg + sa_now + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_apsara_parse_sls_lz4.argtypes = [vp, vp, vp, u64, u8] + sa_cfg + sa_now + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_apsara_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sa_cfg + sa_now + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_apsara_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sa_cfg + sa_now + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_sls_serialize_split_regex_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, u32] + sls_cfg + [i32] + \
        sr_tail + [vp, u64, C.POINTER(u64), vp]
    L.lc_split_regex_parse_sls.argtypes = [vp, vp, vp, u64, u8] + sls_cfg + [i32] + sr_tail + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_regex_parse_sls_lz4.argtypes = [vp, vp, vp, u64, u8] + sls_cfg + [i32] + sr_tail + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_regex_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sls_cfg + [i32] + sr_tail + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_regex_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sls_cfg + [i32] + \
        sr_tail + [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    # the split -> regex -> filter chain: the siblings' arguments with the filter behind time_ns
    L.lc_sls_serialize_split_regex_filter_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, u32] + sls_cfg + \
        [i32] + sr_tail + [vp, vp, u64, C.POINTER(u64), vp]
    L.lc_split_regex_filter_parse_sls.argtypes = [vp, vp, vp, u64, u8] + sls_cfg + [i32] + sr_tail + \
        [vp, vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_regex_filter_parse_sls_lz4.argtypes = [vp, vp, vp, u64, u8] + sls_cfg + [i32] + sr_tail + \
        [vp, vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_regex_filter_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sls_cfg + [i32] + \
        sr_tail + [vp, vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_regex_filter_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sls_cfg + \
        [i32] + sr_tail + [vp, vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    # the split -> regex -> timestamp chain: the siblings' arguments with the timestamp stage behind time_ns
    ts_cfg = [C.c_char_p, u32, vp, C.c_int64, i32, i32]  # tkey, tkey_len, ts, now, discard_interval, enable_ns
    L.lc_split_regex_timestamp_tap_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, u32] + sls_cfg + \
        [i32, C.c_char_p, u32, C.c_char_p, u32, vp, vp]
    L.lc_sls_serialize_split_regex_timestamp_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, u32] + sls_cfg + \
        [i32] + sr_tail + [vp, vp, vp, i32, vp, u64, C.POINTER(u64), vp]
    L.lc_split_regex_timestamp_parse_sls.argtypes = [vp, vp, vp, u64, u8] + sls_cfg + [i32] + sr_tail + ts_cfg + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_regex_timestamp_parse_sls_lz4.argtypes = [vp, vp, vp, u64, u8] + sls_cfg + [i32] + sr_tail + \
        ts_cfg + [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_regex_timestamp_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sls_cfg + \
        [i32] + sr_tail + ts_cfg + [vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_regex_timestamp_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sls_cfg + \
        [i32] + sr_tail + ts_cfg + [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    # the split -> delimiter chain: the delimiter's arguments (sep .. copy_raw), then the split -> regex tail
    sd_cfg = [vp, u32, u8, i32, i32, i32, u32]  # sep .. max_fields of the host-buffer calls
    L.lc_sls_serialize_split_delim_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp, u32, vp, u32, u8,
                                                   i32, i32] + sls_cfg + sr_tail + [vp, u64, C.POINTER(u64), vp]
    L.lc_split_delim_parse_sls.argtypes = [vp, vp, u64, u8] + sd_cfg + sls_cfg + sr_tail + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_delim_parse_sls_lz4.argtypes = [vp, vp, u64, u8] + sd_cfg + sls_cfg + sr_tail + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_delim_parse_sls.argtypes = [vp, vp, u64, vp, vp, vp, i32] + sd_cfg + sls_cfg + sr_tail + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_delim_parse_sls_lz4.argtypes = [vp, vp, u64, vp, vp, vp, i32] + sd_cfg + sls_cfg + \
        sr_tail + [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    # the split -> delimiter -> regex chain: allow_short, max_fields, both stages' arguments, the split -> regex tail
    sdr_cfg = [i32, u32] + chain_cfg + sr_tail
    L.lc_sls_serialize_split_delim_regex_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp, u32] + \
        chain_cfg + sr_tail + [vp, vp, vp, vp, vp, u32, vp, u64, C.POINTER(u64), vp]
    L.lc_split_delim_regex_parse_sls.argtypes = [vp, vp, vp, u64, u8] + sdr_cfg + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_delim_regex_parse_sls_lz4.argtypes = [vp, vp, vp, u64, u8] + sdr_cfg + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_delim_regex_parse_sls.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sdr_cfg + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_delim_regex_parse_sls_lz4.argtypes = [vp, vp, vp, u64, vp, vp, vp, i32] + sdr_cfg + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    # the split -> delimiter -> timestamp chain: the split -> delimiter arguments with the timestamp stage behind time_ns
    L.lc_split_delim_timestamp_tap_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp, u32, vp, u32, u8, i32,
                                                   i32] + sls_cfg + [C.c_char_p, u32, C.c_char_p, u32, vp, u64, vp, vp]
    L.lc_sls_serialize_split_delim_timestamp_dev.argtypes = [vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp, u32, vp, u32,
                                                             u8, i32, i32] + sls_cfg + sr_tail + \
        [vp, vp, vp, i32, vp, u64, C.POINTER(u64), vp]
    L.lc_split_delim_timestamp_parse_sls.argtypes = [vp, vp, u64, u8] + sd_cfg + sls_cfg + sr_tail + sjt_ts + \
        [vp, u64, C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_split_delim_timestamp_parse_sls_lz4.argtypes = [vp, vp, u64, u8] + sd_cfg + sls_cfg + sr_tail + sjt_ts + \
        [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp]
    L.lc_multiline_split_delim_timestamp_parse_sls.argtypes = [vp, vp, u64, vp, vp, vp, i32] + sd_cfg + sls_cfg + \
        sr_tail + sjt_ts + [vp, u64, C.POINTER(u64), C.POINTER(u64), vp, vp]
    L.lc_multiline_split_delim_timestamp_parse_sls_lz4.argtypes = [vp, vp, u64, vp, vp, vp, i32] + sd_cfg + \
        sls_cfg + sr_tail + sjt_ts + [vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), vp, vp]
    _LIB = L
    return L


def version():
    return lib().lc_version().decode()


def device_count():
    return int(lib().lc_device_count())


def _check(rc):
    if rc != LC_OK:
        raise LcError(rc, lib().lc_last_error().decode())


def _p(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(int(a))


def _u8(buf):
    if isinstance(buf, np.ndarray):
        assert buf.dtype == np.uint8 and buf.flags.c_contiguous
        return buf
    return np.frombuffer(bytes(buf), dtype=np.uint8)


class Regex:
    """Compiled pattern (host object; boost::regex(pattern) replacement)."""

    def __init__(self, pattern):
        if isinstance(pattern, str):
            pattern = pattern.encode("utf-8")
        self.pattern = pattern
        h = C.c_void_p()
        L = lib()
        rc = L.lc_regex_compile(pattern, len(pattern), C.byref(h))
        self._h = h
        if rc != LC_OK:
            msg = L.lc_last_error().decode()
            L.lc_regex_free(h)
            self._h = None
            raise LcError(rc, msg)
        self.ngroups = int(L.lc_regex_ngroups(h))
        info = np.zeros(8, np.uint32)
        L.lc_regex_info(h, _p(info))
        self.info = dict(zip(("mode", "classes", "walkers", "ctx", "rev_states", "prefix_states", "table_bytes",
                              "insts"), (int(x) for x in info)))

    def __del__(self):
        try:
            if self._h:
                lib().lc_regex_free(self._h)
        except Exception:
            pass


LC_TS_OK, LC_TS_NOT_FOUND, LC_TS_FAILED, LC_TS_DISCARDED = 0, 1, 2, 3
LC_TS_NO_KEY = 0xFFFFFFFF


class Timestamp:
    """Compiled SourceFormat of ProcessorParseTimestampNative (lc_timestamp_compile): SourceYear (-1 unset, 0 deduce,
    > 0 that year) and the timezone adjustment (mLogTimeZoneOffsetSecond) are fixed here, and so is the process's
    local zone."""

    def __init__(self, fmt, source_year=-1, tz_adjust=0):
        if isinstance(fmt, str):
            fmt = fmt.encode("utf-8")
        self.format = fmt
        h = C.c_void_p()
        L = lib()
        rc = L.lc_timestamp_compile(fmt, len(fmt), int(source_year), int(tz_adjust), C.byref(h))
        self._h = h
        if rc != LC_OK:
            self._h = None
            raise LcError(rc, L.lc_last_error().decode())

    def __del__(self):
        try:
            if self._h:
                lib().lc_timestamp_free(self._h)
        except Exception:
            pass


class Apsara:
    """ProcessorParseApsaraNative's Init (lc_apsara_compile): SourceKey and the timezone adjustment
    (mLogTimeZoneOffsetSecond) are fixed here, and so is the process's local zone."""

    def __init__(self, source_key, tz_adjust=0):
        if isinstance(source_key, str):
            source_key = source_key.encode("utf-8")
        h = C.c_void_p()
        L = lib()
        rc = L.lc_apsara_compile(source_key, len(source_key), int(tz_adjust), C.byref(h))
        self._h = h
        if rc != LC_OK:
            self._h = None
            raise LcError(rc, L.lc_last_error().decode())

    def __del__(self):
        try:
            if self._h:
                lib().lc_apsara_free(self._h)
        except Exception:
            pass


# lc_apsara_parse's status values and base-field keys
LC_APSARA_OK, LC_APSARA_NOT_FOUND, LC_APSARA_EMPTY, LC_APSARA_FAILED, LC_APSARA_DISCARDED = 0, 1, 2, 3, 4
LC_APSARA_OVERWRITTEN = 0x80
LC_APSARA_KEY_LEVEL = 0xFFFFFFF0
APSARA_BASE_KEYS = (b"__LEVEL__", b"__THREAD__", b"__FILE__", b"__LINE__")


class Json:
    """ProcessorParseJsonNative's Init (lc_json_compile): SourceKey is fixed here."""

    def __init__(self, source_key):
        if isinstance(source_key, str):
            source_key = source_key.encode("utf-8")
        h = C.c_void_p()
        L = lib()
        rc = L.lc_json_compile(source_key, len(source_key), C.byref(h))
        self._h = h
        if rc != LC_OK:
            self._h = None
            raise LcError(rc, L.lc_last_error().decode())

    def __del__(self):
        try:
            if self._h:
                lib().lc_json_free(self._h)
        except Exception:
            pass


# lc_json_parse's status values and arena tag
LC_JSON_OK, LC_JSON_NOT_FOUND, LC_JSON_EMPTY, LC_JSON_FAILED, LC_JSON_OVERWRITTEN = 0, 1, 2, 3, 0x80
LC_JSON_ARENA = 0x80000000
LC_ERR_INTERNAL = 7


def _rh(r):
    return r._h if r is not None else None


LC_FILTER_NOT, LC_FILTER_AND, LC_FILTER_OR = 0xFFFFFFFD, 0xFFFFFFFE, 0xFFFFFFFF
_FILTER_OPS = {"not": LC_FILTER_NOT, "and": LC_FILTER_AND, "or": LC_FILTER_OR}


class _FilterDesc(C.Structure):
    _fields_ = [("nleaves", C.c_uint32), ("keys", C.c_void_p), ("key_lens", C.c_void_p), ("regs", C.c_void_p),
                ("nprog", C.c_uint32), ("prog", C.c_void_p)]


class Filter:
    """A processor_filter_regex_native rule as the split -> regex -> filter calls take it (lc_filter_desc_t).
    leaves: [(key bytes, Regex or None)]; prog: postfix program, each entry a leaf index or "not" / "and" / "or" (or
    the LC_FILTER_* codes, or any int, to exercise the refusals).  An empty prog is BYPASS mode."""

    def __init__(self, leaves, prog):
        self.leaves = list(leaves)
        self._karr = (C.c_char_p * max(len(self.leaves), 1))(*[k for k, _ in self.leaves])
        self._kl = np.array([len(k) for k, _ in self.leaves] or [0], np.uint32)
        self._regs = (C.c_void_p * max(len(self.leaves), 1))(*[_rh(r) for _, r in self.leaves])
        self._prog = np.array([_FILTER_OPS[x] if isinstance(x, str) else x for x in prog] or [0], np.uint32)
        self.desc = _FilterDesc(len(self.leaves), C.cast(self._karr, C.c_void_p), _p(self._kl),
                                C.cast(self._regs, C.c_void_p), len(prog), _p(self._prog))

    @staticmethod
    def rule(pairs):
        """RULE mode: every (key, Regex) must hold"""
        prog = [0] if pairs else []
        for i in range(1, len(pairs)):
            prog += [i, "and"]
        return Filter(pairs, prog)

    def ptr(self):
        return C.cast(C.pointer(self.desc), C.c_void_p)


class Engine:
    """One engine per (GPU, host thread)."""

    def __init__(self, device=0):
        h = C.c_void_p()
        _check(lib().lc_engine_create(device, C.byref(h)))
        self._h = h
        self.device = device

    def close(self):
        if self._h:
            lib().lc_engine_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        _check(lib().lc_engine_sync(self._h))

    @property
    def stream(self):
        return int(lib().lc_engine_stream(self._h) or 0)

    @property
    def launches(self):
        return int(lib().lc_engine_launch_count(self._h))

    # ---- host-buffer API ---------------------------------------------------------------------
    def split_lines(self, buf, split_char=10, cap=None):
        a = _u8(buf)
        cap = int(cap if cap is not None else max(1, a.size))
        off = np.empty(cap, np.uint32)
        ln = np.empty(cap, np.uint32)
        n = C.c_uint64(0)
        _check(lib().lc_split_lines(self._h, _p(a), a.size, split_char, _p(off), _p(ln), cap, C.byref(n)))
        return off[:n.value], ln[:n.value]

    def regex_parse(self, rx, base, ev_off, ev_len, nkeys):
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        n, G = ev_off.size, rx.ngroups
        status = np.empty(n, np.uint8)
        co = np.empty((n, G), np.uint32)
        cl = np.empty((n, G), np.uint32)
        _check(lib().lc_regex_parse(self._h, rx._h, _p(a), a.size, _p(ev_off), _p(ev_len), n, nkeys, _p(status),
                                    _p(co), _p(cl)))
        return status, co, cl

    @staticmethod
    def _multi_handles(rxs, nkeys):
        arr = (C.c_void_p * len(rxs))(*[r._h.value if isinstance(r._h, C.c_void_p) else r._h for r in rxs])
        nk = np.ascontiguousarray(nkeys, np.uint32)
        assert nk.size == len(rxs)
        return arr, nk

    def regex_parse_multi(self, rxs, nkeys, base, ev_off, ev_len, sel=None, row_pitch=None):
        """First-match-wins over several patterns in one grid; returns (which, status, cap_off, cap_len)."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        n = ev_off.size
        G = int(row_pitch if row_pitch is not None else max(r.ngroups for r in rxs))
        arr, nk = self._multi_handles(rxs, nkeys)
        which = np.empty(n, np.uint8)
        status = np.empty(n, np.uint8)
        co = np.empty((n, G), np.uint32)
        cl = np.empty((n, G), np.uint32)
        if sel is not None:
            sel = np.ascontiguousarray(sel, np.uint8)
        _check(lib().lc_regex_parse_multi(self._h, arr, len(rxs), _p(nk), _p(a), a.size, _p(ev_off), _p(ev_len), n,
                                          _p(sel), _p(which), _p(status), G, _p(co), _p(cl)))
        return which, status, co, cl

    def regex_parse_multi_dev(self, rxs, nkeys, d_base, base_len, d_ev_off, d_ev_len, n, d_sel, d_which, d_status,
                              row_pitch, d_cap_off, d_cap_len):
        arr, nk = self._multi_handles(rxs, nkeys)
        _check(lib().lc_regex_parse_multi_dev(self._h, arr, len(rxs), _p(nk), _p(d_base), base_len, _p(d_ev_off),
                                              _p(d_ev_len), n, _p(d_sel), _p(d_which), _p(d_status), row_pitch,
                                              _p(d_cap_off), _p(d_cap_len)))

    def regex_parse_strided_dev(self, rx, d_base, base_len, d_ev_off, d_ev_len, ev_stride, n, nkeys, d_status,
                                d_cap_off, d_cap_len):
        _check(lib().lc_regex_parse_strided_dev(self._h, rx._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len),
                                                ev_stride, n, nkeys, _p(d_status), _p(d_cap_off), _p(d_cap_len)))

    def set_stream(self, stream):
        _check(lib().lc_engine_set_stream(self._h, _p(stream) if stream else None))

    def remove_last_incomplete_log(self, buf, start, end, allow_rollback=True):
        """LogFileReader::RemoveLastIncompleteLog (raw text) -> (bytes to keep, rollbackLineFeedCount)."""
        a = _u8(buf)
        keep, rb = C.c_uint64(0), C.c_int32(0)
        _check(lib().lc_remove_last_incomplete_log(self._h, _p(a), a.size, _rh(start), _rh(end),
                                                   int(bool(allow_rollback)), C.byref(keep), C.byref(rb)))
        return int(keep.value), int(rb.value)

    def regex_prefix_match(self, rx, base, ev_off, ev_len):
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        out = np.empty(ev_off.size, np.uint8)
        _check(lib().lc_regex_prefix_match(self._h, rx._h, _p(a), a.size, _p(ev_off), _p(ev_len), ev_off.size,
                                           _p(out)))
        return out.astype(bool)

    def regex_match(self, rx, base, ev_off, ev_len):
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        out = np.empty(ev_off.size, np.uint8)
        _check(lib().lc_regex_match(self._h, rx._h, _p(a), a.size, _p(ev_off), _p(ev_len), ev_off.size, _p(out)))
        return out.astype(bool)

    def multiline_split(self, buf, start, cont, end, discard, cap=None):
        a = _u8(buf)
        cap = int(cap if cap is not None else max(1, a.size))
        off = np.empty(cap, np.uint32)
        ln = np.empty(cap, np.uint32)
        fl = np.empty(cap, np.uint8)
        ctr = np.zeros(3, np.uint64)
        n = C.c_uint64(0)
        _check(lib().lc_multiline_split(self._h, _p(a), a.size, _rh(start), _rh(cont), _rh(end), int(bool(discard)),
                                        _p(off), _p(ln), _p(fl), cap, C.byref(n), _p(ctr)))
        return off[:n.value], ln[:n.value], fl[:n.value], ctr

    def delim_parse(self, base, ev_off, ev_len, sep: bytes, quote: int, nkeys, extend, allow_short, max_fields):
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        n = ev_off.size
        status = np.empty(n, np.uint8)
        nf = np.empty(n, np.uint32)
        fo = np.empty((n, max_fields), np.uint32)
        fl = np.empty((n, max_fields), np.uint32)
        fd = np.empty((n, max_fields), np.uint32)
        sp = np.frombuffer(sep, np.uint8)
        _check(lib().lc_delim_parse(self._h, _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(sp), len(sep), quote, nkeys,
                                    int(bool(extend)), int(bool(allow_short)), max_fields, _p(status), _p(nf), _p(fo),
                                    _p(fl), _p(fd)))
        return status, nf, fo, fl, fd

    # ---- device-pointer API (ints = device addresses) ---------------------------------------------
    def sls_serialize_logs(self, events, enable_ns=True):
        """events: list of (time, ns or None, [(key bytes, value bytes), ...]) -> the LogGroup's `Logs` fields (bytes).
        Packs the keys and values into one arena the way LogEvent contents alias the SourceBuffer."""
        arena = bytearray()
        koff, klen, voff, vlen, begin, times, nss = [], [], [], [], [0], [], []
        for t, ns, contents in events:
            for k, v in contents:
                koff.append(len(arena))
                klen.append(len(k))
                arena += k
                voff.append(len(arena))
                vlen.append(len(v))
                arena += v
            begin.append(len(koff))
            times.append(int(t) & 0xFFFFFFFF)
            nss.append(0xFFFFFFFF if (ns is None or not enable_ns) else int(ns))
        n = len(times)
        base = np.frombuffer(bytes(arena), np.uint8) if arena else np.zeros(1, np.uint8)
        a32 = lambda x: np.array(x if x else [0], np.uint32)  # noqa: E731
        need = C.c_uint64(0)
        cap = len(arena) + 32 * len(koff) + 16 * n + 64
        out = np.zeros(max(cap, 1), np.uint8)
        _check(lib().lc_sls_serialize_logs(self._h, _p(base), len(arena), n, _p(a32(times)), _p(a32(nss)),
                                           _p(np.array(begin, np.uint64)), _p(a32(koff)), _p(a32(klen)),
                                           _p(a32(voff)), _p(a32(vlen)), _p(out), cap, C.byref(need)))
        return bytes(out[:need.value])

    def sls_serialize_parsed_dev(self, d_base, base_len, d_ev_off, d_ev_len, d_status, d_cap_off, d_cap_len, row_pitch,
                                 n, keys, fail_key, d_ev_time, d_ev_time_ns, d_out, out_cap):
        """keys: list of bytes; fail_key: bytes or None.  Returns the number of wire bytes written to d_out."""
        arr = (C.c_char_p * max(len(keys), 1))(*keys)
        kl = np.array([len(k) for k in keys] or [0], np.uint32)
        need = C.c_uint64(0)
        _check(lib().lc_sls_serialize_parsed_dev(self._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len),
                                                 _p(d_status), _p(d_cap_off), _p(d_cap_len), row_pitch, n, arr, _p(kl),
                                                 len(keys), fail_key, len(fail_key) if fail_key else 0, _p(d_ev_time),
                                                 _p(d_ev_time_ns), _p(d_out), out_cap, C.byref(need)))
        return int(need.value)

    @staticmethod
    def _delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw):
        """keys / source_key / renamed_key: bytes (renamed_key None = source_key); returns the C arguments"""
        arr = (C.c_char_p * max(len(keys), 1))(*keys)
        kl = np.array([len(k) for k in keys] or [0], np.uint32)
        rk = source_key if renamed_key is None else renamed_key
        return (arr, kl), [C.cast(arr, C.c_void_p), _p(kl), len(keys), source_key, len(source_key), rk, len(rk),
                           int(bool(keep_fail)), int(bool(keep_succeed)), int(bool(copy_raw))]

    def sls_serialize_delim_dev(self, d_base, base_len, d_ev_off, d_ev_len, n, d_status, d_nf, d_fo, d_fl, d_fd,
                                max_fields, sep: bytes, quote, treatment, keys, source_key, renamed_key=None,
                                keep_fail=False, keep_succeed=False, copy_raw=False, d_ev_time=None,
                                d_ev_time_ns=None, d_out=None, out_cap=0):
        """Wire bytes of the events ProcessorParseDelimiterNative leaves behind, from the device tables of one
        delim_parse_dev call (treatment: "extend" / "keep" / "discard").  Returns the byte count written to d_out, or
        with d_out None the byte count needed."""
        sp = np.frombuffer(sep, np.uint8)
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        need = C.c_uint64(0)
        rc = lib().lc_sls_serialize_delim_dev(self._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len), n,
                                              _p(d_status), _p(d_nf), _p(d_fo), _p(d_fl), _p(d_fd), max_fields, _p(sp),
                                              len(sep), quote, int(treatment == "extend"), int(treatment == "discard"),
                                              *cfg, _p(d_ev_time), _p(d_ev_time_ns), _p(d_out), out_cap, C.byref(need))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value)  # a sizing query
        _check(rc)
        return int(need.value)

    def delim_parse_sls(self, base, ev_off, ev_len, ev_time, sep: bytes, quote, treatment, keys, source_key,
                        renamed_key=None, keep_fail=False, keep_succeed=False, copy_raw=False, allow_short=True,
                        max_fields=None, ev_time_ns=None, out_cap=None):
        """Host buffers in, wire bytes out (lc_delim_parse_sls).  Returns (bytes, counters[4] = successful, failed,
        discarded, blank).  Without out_cap the output is sized by a first estimate and, if short, the exact size."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        t = np.ascontiguousarray(ev_time, np.uint32)
        ns = None if ev_time_ns is None else np.ascontiguousarray(ev_time_ns, np.uint32)
        n = ev_off.size
        mf = int(max_fields if max_fields is not None else len(keys) + 16)
        sp = np.frombuffer(sep, np.uint8)
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        cap = int(out_cap if out_cap is not None else 2 * a.size + 64 * n + 64)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need = C.c_uint64(0)
            ctr = np.zeros(4, np.uint64)
            rc = lib().lc_delim_parse_sls(self._h, _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(t), _p(ns), _p(sp),
                                          len(sep), quote, int(treatment == "extend"), int(treatment == "discard"),
                                          int(bool(allow_short)), mf, *cfg, _p(out), cap, C.byref(need), _p(ctr))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), ctr
        _check(rc)

    def sls_serialize_regex_dev(self, d_base, base_len, d_ev_off, d_ev_len, n, d_status, d_cap_off, d_cap_len,
                                row_pitch, keys, source_key, renamed_key=None, keep_fail=False, keep_succeed=False,
                                copy_raw=False, whole_line=False, d_ev_time=None, d_ev_time_ns=None, d_out=None,
                                out_cap=0):
        """Wire bytes of the events ProcessorParseRegexNative leaves behind, from the device tables of one
        regex_parse_dev call (d_status / d_cap_* may be None in whole-line mode).  Returns (byte count written to d_out,
        counters[3] = successful, failed, discarded); with d_out None the byte count needed."""
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        need = C.c_uint64(0)
        ctr = np.zeros(3, np.uint64)
        rc = lib().lc_sls_serialize_regex_dev(self._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len), n,
                                              _p(d_status), _p(d_cap_off), _p(d_cap_len), row_pitch, *cfg,
                                              int(bool(whole_line)), _p(d_ev_time), _p(d_ev_time_ns), _p(d_out),
                                              out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def regex_parse_sls(self, rx, base, ev_off, ev_len, ev_time, keys, source_key, renamed_key=None, keep_fail=False,
                        keep_succeed=False, copy_raw=False, whole_line=False, ev_time_ns=None, out_cap=None):
        """Host buffers in, wire bytes out (lc_regex_parse_sls; rx may be None in whole-line mode).  Returns (bytes,
        counters[3] = successful, failed, discarded).  Without out_cap the output is sized by a first estimate and,
        if short, the exact size."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        t = np.ascontiguousarray(ev_time, np.uint32)
        ns = None if ev_time_ns is None else np.ascontiguousarray(ev_time_ns, np.uint32)
        n = ev_off.size
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        cap = int(out_cap if out_cap is not None else 2 * a.size + 64 * n + 64)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need = C.c_uint64(0)
            ctr = np.zeros(3, np.uint64)
            rc = lib().lc_regex_parse_sls(self._h, _rh(rx), _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(t), _p(ns),
                                          *cfg, int(bool(whole_line)), _p(out), cap, C.byref(need), _p(ctr))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), ctr
        _check(rc)

    @staticmethod
    def _sls_lz4(call, nctr, tail, out_cap, est):
        """runs call(tail, out, cap, &need, &raw, ctr) of a fused LZ4 call, sized by est first and by the exact block
        size when that was short; returns (block, raw_len, counters)"""
        tl = np.frombuffer(bytes(tail), np.uint8)
        cap = int(out_cap if out_cap is not None else est + est // 255 + 16)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need, raw = C.c_uint64(0), C.c_uint64(0)
            ctr = np.zeros(nctr, np.uint64)
            rc = call(_p(tl) if tl.size else None, tl.size, _p(out), cap, C.byref(need), C.byref(raw), _p(ctr))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), int(raw.value), ctr
        _check(rc)

    def regex_parse_sls_lz4(self, rx, base, ev_off, ev_len, ev_time, keys, source_key, renamed_key=None,
                            keep_fail=False, keep_succeed=False, copy_raw=False, whole_line=False, ev_time_ns=None,
                            tail=b"", out_cap=None):
        """regex_parse_sls's records followed by `tail` (the group-level fields) as ONE LZ4 block
        (lc_regex_parse_sls_lz4).  Returns (block, raw_len, counters[3])."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        t = np.ascontiguousarray(ev_time, np.uint32)
        ns = None if ev_time_ns is None else np.ascontiguousarray(ev_time_ns, np.uint32)
        n = ev_off.size
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        return self._sls_lz4(
            lambda *rest: lib().lc_regex_parse_sls_lz4(self._h, _rh(rx), _p(a), a.size, _p(ev_off), _p(ev_len), n,
                                                       _p(t), _p(ns), *cfg, int(bool(whole_line)), *rest),
            3, tail, out_cap, 2 * a.size + 64 * n + 64 + len(tail))

    def delim_parse_sls_lz4(self, base, ev_off, ev_len, ev_time, sep: bytes, quote, treatment, keys, source_key,
                            renamed_key=None, keep_fail=False, keep_succeed=False, copy_raw=False, allow_short=True,
                            max_fields=None, ev_time_ns=None, tail=b"", out_cap=None):
        """delim_parse_sls's records followed by `tail` (the group-level fields) as ONE LZ4 block
        (lc_delim_parse_sls_lz4).  Returns (block, raw_len, counters[4])."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        t = np.ascontiguousarray(ev_time, np.uint32)
        ns = None if ev_time_ns is None else np.ascontiguousarray(ev_time_ns, np.uint32)
        n = ev_off.size
        mf = int(max_fields if max_fields is not None else len(keys) + 16)
        sp = np.frombuffer(sep, np.uint8)
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        return self._sls_lz4(
            lambda *rest: lib().lc_delim_parse_sls_lz4(self._h, _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(t),
                                                       _p(ns), _p(sp), len(sep), quote, int(treatment == "extend"),
                                                       int(treatment == "discard"), int(bool(allow_short)), mf, *cfg,
                                                       *rest),
            4, tail, out_cap, 2 * a.size + 64 * n + 64 + len(tail))

    @staticmethod
    def _chain_cfg(delim, regex):
        """the C arguments of a delimiter -> regex chain.  delim: dict(sep, quote, treatment, keys, source_key,
        renamed_key=None, keep_fail=False, keep_succeed=False, copy_raw=False); regex: dict(keys, source_key,
        renamed_key=None, keep_fail=False, keep_succeed=False, copy_raw=False, whole_line=False); keys as bytes."""
        sp = np.frombuffer(delim["sep"], np.uint8)
        dk, dcfg = Engine._delim_sls_cfg(delim["keys"], delim["source_key"], delim.get("renamed_key"),
                                         delim.get("keep_fail"), delim.get("keep_succeed"), delim.get("copy_raw"))
        rk, rcfg = Engine._delim_sls_cfg(regex["keys"], regex["source_key"], regex.get("renamed_key"),
                                         regex.get("keep_fail"), regex.get("keep_succeed"), regex.get("copy_raw"))
        tr = delim["treatment"]
        return (sp, dk, rk), [_p(sp), sp.size, delim["quote"], int(tr == "extend"), int(tr == "discard")] + dcfg + \
            rcfg + [int(bool(regex.get("whole_line")))]

    def delim_regex_tap_dev(self, d_base, base_len, base_cap, d_ev_off, d_ev_len, n, d_status, d_nf, d_fo, d_fl, d_fd,
                            max_fields, delim, regex, d_val_off, d_val_len):
        """The regex stage's event table of a delimiter -> regex chain (lc_delim_regex_tap_dev) into d_val_off /
        d_val_len, side copies behind base_len in d_base (capacity base_cap).  Returns the side bytes; raises
        LcError(LC_ERR_CAPACITY) when they do not fit (nothing written; .need = the side bytes)."""
        _keep, cfg = self._chain_cfg(delim, regex)
        side = C.c_uint64(0)
        rc = lib().lc_delim_regex_tap_dev(self._h, _p(d_base), base_len, base_cap, _p(d_ev_off), _p(d_ev_len), n,
                                          _p(d_status), _p(d_nf), _p(d_fo), _p(d_fl), _p(d_fd), max_fields, *cfg,
                                          _p(d_val_off), _p(d_val_len), C.byref(side))
        if rc != LC_OK:
            err = LcError(rc, lib().lc_last_error().decode())
            err.need = int(side.value)
            raise err
        return int(side.value)

    def sls_serialize_delim_regex_dev(self, d_base, base_len, d_ev_off, d_ev_len, n, d_status, d_nf, d_fo, d_fl, d_fd,
                                      max_fields, delim, regex, d_val_off, d_val_len, d_re_status, d_cap_off,
                                      d_cap_len, row_pitch, d_ev_time, d_ev_time_ns=None, d_out=None, out_cap=0):
        """Wire bytes of a delimiter -> regex chain from device tables (lc_sls_serialize_delim_regex_dev).  Returns
        (byte count written to d_out, counters[8]); with d_out None the byte count needed."""
        _keep, cfg = self._chain_cfg(delim, regex)
        need = C.c_uint64(0)
        ctr = np.zeros(8, np.uint64)
        rc = lib().lc_sls_serialize_delim_regex_dev(self._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len), n,
                                                    _p(d_status), _p(d_nf), _p(d_fo), _p(d_fl), _p(d_fd), max_fields,
                                                    *cfg, _p(d_val_off), _p(d_val_len), _p(d_re_status), _p(d_cap_off),
                                                    _p(d_cap_len), row_pitch, _p(d_ev_time), _p(d_ev_time_ns),
                                                    _p(d_out), out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def _chain_host(self, rx, base, ev_off, ev_len, ev_time, ev_time_ns, allow_short, max_fields, delim, regex):
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        t = np.ascontiguousarray(ev_time, np.uint32)
        ns = None if ev_time_ns is None else np.ascontiguousarray(ev_time_ns, np.uint32)
        n = ev_off.size
        mf = int(max_fields if max_fields is not None else len(delim["keys"]) + 16)
        keep, cfg = self._chain_cfg(delim, regex)
        head = [self._h, _rh(rx), _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(t), _p(ns), int(bool(allow_short)), mf]
        return (a, ev_off, ev_len, t, ns, keep), head + cfg, 2 * a.size + 96 * n + 64

    def delim_regex_parse_sls(self, rx, base, ev_off, ev_len, ev_time, delim, regex, allow_short=True,
                              max_fields=None, ev_time_ns=None, out_cap=None):
        """Host buffers in, wire bytes of the delimiter -> regex chain out (lc_delim_regex_parse_sls; rx may be None
        in whole-line mode).  Returns (bytes, counters[8])."""
        _keep, args, est = self._chain_host(rx, base, ev_off, ev_len, ev_time, ev_time_ns, allow_short, max_fields,
                                            delim, regex)
        cap = int(out_cap if out_cap is not None else est)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need = C.c_uint64(0)
            ctr = np.zeros(8, np.uint64)
            rc = lib().lc_delim_regex_parse_sls(*args, _p(out), cap, C.byref(need), _p(ctr))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), ctr
        _check(rc)

    def delim_regex_parse_sls_lz4(self, rx, base, ev_off, ev_len, ev_time, delim, regex, allow_short=True,
                                  max_fields=None, ev_time_ns=None, tail=b"", out_cap=None):
        """delim_regex_parse_sls's records followed by `tail` as ONE LZ4 block (lc_delim_regex_parse_sls_lz4).
        Returns (block, raw_len, counters[8])."""
        _keep, args, est = self._chain_host(rx, base, ev_off, ev_len, ev_time, ev_time_ns, allow_short, max_fields,
                                            delim, regex)
        return self._sls_lz4(lambda *rest: lib().lc_delim_regex_parse_sls_lz4(*args, *rest), 8, tail, out_cap,
                             est + len(tail))

    @staticmethod
    def _span_keys(key, offset_key, src_pos, time, time_ns):
        """key / offset_key: bytes (offset_key None = no offset key); time_ns None = no Time_ns"""
        return [key, len(key), offset_key, len(offset_key) if offset_key is not None else 0, int(src_pos),
                int(time) & 0xFFFFFFFF, 0xFFFFFFFF if time_ns is None else int(time_ns)]

    def sls_serialize_spans_dev(self, d_src, src_len, d_off, d_len, n, key, offset_key=None, src_pos=0, time=0,
                                time_ns=None, d_out=None, out_cap=0):
        """Wire bytes of the events a splitter cuts from one source value, from the device piece tables of one
        split_lines_dev / multiline_split_dev call (lc_sls_serialize_spans_dev).  Returns the byte count written to
        d_out, or with d_out None the byte count needed."""
        need = C.c_uint64(0)
        rc = lib().lc_sls_serialize_spans_dev(self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n,
                                              *self._span_keys(key, offset_key, src_pos, time, time_ns), _p(d_out),
                                              out_cap, C.byref(need))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value)  # a sizing query
        _check(rc)
        return int(need.value)

    def _split_sls(self, fn, buf, extra, key, offset_key, src_pos, time, time_ns, out_cap, tail):
        a = _u8(buf)
        cap = int(out_cap if out_cap is not None else 2 * a.size + 4096)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need, nev = C.c_uint64(0), C.c_uint64(0)
            for t in tail:
                t[:] = 0  # (the counters are added to: a second, exactly sized call starts again from zero)
            rc = fn(self._h, _p(a), a.size, *extra, *self._span_keys(key, offset_key, src_pos, time, time_ns), _p(out),
                    cap, C.byref(need), C.byref(nev), *(_p(t) for t in tail))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), int(nev.value)
        _check(rc)

    def split_sls(self, buf, split_char, key, offset_key=None, src_pos=0, time=0, time_ns=None, out_cap=None):
        """Host source value in, wire bytes out (lc_split_sls).  Returns (bytes, number of pieces)."""
        return self._split_sls(lib().lc_split_sls, buf, [split_char], key, offset_key, src_pos, time, time_ns, out_cap,
                               [])

    def multiline_split_sls(self, buf, start, cont, end, discard, key, offset_key=None, src_pos=0, time=0,
                            time_ns=None, out_cap=None):
        """Host source value in, wire bytes out (lc_multiline_split_sls).  Returns (bytes, number of events,
        counters[3] = matched_events, input_lines, unmatched_lines)."""
        ctr = np.zeros(3, np.uint64)
        data, nev = self._split_sls(lib().lc_multiline_split_sls, buf,
                                    [_rh(start), _rh(cont), _rh(end), int(bool(discard))], key, offset_key, src_pos,
                                    time, time_ns, out_cap, [ctr])
        return data, nev, ctr

    @staticmethod
    def _sr_tail(offset_key, src_pos, time, time_ns):
        """offset_key: bytes, None = no log.file.offset metadata; time_ns None = no Time_ns"""
        return [offset_key, len(offset_key) if offset_key is not None else 0, int(src_pos), int(time) & 0xFFFFFFFF,
                0xFFFFFFFF if time_ns is None else int(time_ns)]

    def sls_serialize_split_regex_dev(self, d_src, src_len, d_off, d_len, n, d_status, d_cap_off, d_cap_len,
                                      row_pitch, keys, source_key, renamed_key=None, keep_fail=False,
                                      keep_succeed=False, copy_raw=False, whole_line=False, offset_key=None,
                                      src_pos=0, time=0, time_ns=None, d_out=None, out_cap=0):
        """Wire bytes of the split -> regex chain from the device piece tables of one split_lines_dev /
        multiline_split_dev call and the device tables of regex_parse_dev over those pieces
        (lc_sls_serialize_split_regex_dev).  Returns (byte count written to d_out, counters[3] = successful, failed,
        discarded); with d_out None the byte count needed."""
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        need = C.c_uint64(0)
        ctr = np.zeros(3, np.uint64)
        rc = lib().lc_sls_serialize_split_regex_dev(self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n,
                                                    _p(d_status), _p(d_cap_off), _p(d_cap_len), row_pitch, *cfg,
                                                    int(bool(whole_line)),
                                                    *self._sr_tail(offset_key, src_pos, time, time_ns), _p(d_out),
                                                    out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def _split_regex(self, fn, rx, buf, extra, keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw,
                     whole_line, offset_key, src_pos, time, time_ns, out_cap, ml, tail, filt=None, tsx=None):
        """one host-buffer split -> regex call, sized by an estimate first and by the exact size when that was short;
        tail None: the wire bytes, else records ‖ tail as one LZ4 block.  filt (a Filter): the _filter_ call, with
        counters[4]; tsx (_ts_args): the _timestamp_ call, with counters[8].  Returns (bytes, raw_len, n_events,
        counters[3], [4] or [8], ml_counters[3] or None)"""
        a = _u8(buf)
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        tl = None if tail is None else np.frombuffer(bytes(tail), np.uint8)
        est = 2 * a.size + 4096 + (0 if tl is None else tl.size)
        cap = int(out_cap if out_cap is not None else est + est // 255 + 16)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
            ctr, mctr = np.zeros(8 if tsx else 3 if filt is None else 4, np.uint64), np.zeros(3, np.uint64)
            z = [] if tl is None else [_p(tl) if tl.size else None, tl.size]
            outs = [_p(out), cap, C.byref(need)] + ([] if tl is None else [C.byref(raw)]) + [C.byref(nev), _p(ctr)]
            f = ([] if filt is None else [filt.ptr()]) + (tsx or [])
            rc = fn(self._h, _rh(rx), _p(a), a.size, *extra, *cfg, int(bool(whole_line)),
                    *self._sr_tail(offset_key, src_pos, time, time_ns), *f, *z, *outs, *([_p(mctr)] if ml else []))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), int(raw.value), int(nev.value), ctr, (mctr if ml else None)
        _check(rc)

    def split_regex_parse_sls(self, rx, buf, split_char, keys, source_key, renamed_key=None, keep_fail=False,
                              keep_succeed=False, copy_raw=False, whole_line=False, offset_key=None, src_pos=0,
                              time=0, time_ns=None, out_cap=None):
        """Host source value in: split, regex (rx may be None in whole-line mode), wire bytes out
        (lc_split_regex_parse_sls).  Returns (bytes, number of pieces, counters[3])."""
        data, _raw, nev, ctr, _m = self._split_regex(
            lib().lc_split_regex_parse_sls, rx, buf, [split_char], keys, source_key, renamed_key, keep_fail,
            keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, False, None)
        return data, nev, ctr

    def split_regex_parse_sls_lz4(self, rx, buf, split_char, keys, source_key, renamed_key=None, keep_fail=False,
                                  keep_succeed=False, copy_raw=False, whole_line=False, offset_key=None, src_pos=0,
                                  time=0, time_ns=None, tail=b"", out_cap=None):
        """split_regex_parse_sls's records followed by `tail` as ONE LZ4 block (lc_split_regex_parse_sls_lz4).
        Returns (block, raw_len, number of pieces, counters[3])."""
        data, raw, nev, ctr, _m = self._split_regex(
            lib().lc_split_regex_parse_sls_lz4, rx, buf, [split_char], keys, source_key, renamed_key, keep_fail,
            keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, False, tail)
        return data, raw, nev, ctr

    def multiline_split_regex_parse_sls(self, rx, buf, start, cont, end, discard, keys, source_key, renamed_key=None,
                                        keep_fail=False, keep_succeed=False, copy_raw=False, whole_line=False,
                                        offset_key=None, src_pos=0, time=0, time_ns=None, out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_regex_parse_sls).  Returns (bytes, number of
        events, counters[3], splitter counters[3] = matched_events, input_lines, unmatched_lines)."""
        data, _raw, nev, ctr, mctr = self._split_regex(
            lib().lc_multiline_split_regex_parse_sls, rx, buf, [_rh(start), _rh(cont), _rh(end), int(bool(discard))],
            keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw, whole_line, offset_key, src_pos, time,
            time_ns, out_cap, True, None)
        return data, nev, ctr, mctr

    def multiline_split_regex_parse_sls_lz4(self, rx, buf, start, cont, end, discard, keys, source_key,
                                            renamed_key=None, keep_fail=False, keep_succeed=False, copy_raw=False,
                                            whole_line=False, offset_key=None, src_pos=0, time=0, time_ns=None,
                                            tail=b"", out_cap=None):
        """multiline_split_regex_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_regex_parse_sls_lz4).  Returns (block, raw_len, number of events, counters[3], splitter
        counters[3])."""
        return self._split_regex(
            lib().lc_multiline_split_regex_parse_sls_lz4, rx, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], keys, source_key, renamed_key, keep_fail,
            keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, True, tail)

    def sls_serialize_split_regex_filter_dev(self, d_src, src_len, d_off, d_len, n, d_status, d_cap_off, d_cap_len,
                                             row_pitch, keys, source_key, filt, renamed_key=None, keep_fail=False,
                                             keep_succeed=False, copy_raw=False, whole_line=False, offset_key=None,
                                             src_pos=0, time=0, time_ns=None, d_out=None, out_cap=0):
        """sls_serialize_split_regex_dev with the Filter filt behind the regex stage
        (lc_sls_serialize_split_regex_filter_dev).  Returns (byte count, counters[4] = successful, failed, discarded,
        removed by the filter); with d_out None the byte count needed."""
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        need = C.c_uint64(0)
        ctr = np.zeros(4, np.uint64)
        rc = lib().lc_sls_serialize_split_regex_filter_dev(self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n,
                                                           _p(d_status), _p(d_cap_off), _p(d_cap_len), row_pitch,
                                                           *cfg, int(bool(whole_line)),
                                                           *self._sr_tail(offset_key, src_pos, time, time_ns),
                                                           filt.ptr(), _p(d_out), out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def split_regex_filter_parse_sls(self, rx, buf, split_char, keys, source_key, filt, renamed_key=None,
                                     keep_fail=False, keep_succeed=False, copy_raw=False, whole_line=False,
                                     offset_key=None, src_pos=0, time=0, time_ns=None, out_cap=None):
        """split_regex_parse_sls with the Filter filt (lc_split_regex_filter_parse_sls).  Returns (bytes, number of
        pieces, counters[4])."""
        data, _raw, nev, ctr, _m = self._split_regex(
            lib().lc_split_regex_filter_parse_sls, rx, buf, [split_char], keys, source_key, renamed_key, keep_fail,
            keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, False, None, filt)
        return data, nev, ctr

    def split_regex_filter_parse_sls_lz4(self, rx, buf, split_char, keys, source_key, filt, renamed_key=None,
                                         keep_fail=False, keep_succeed=False, copy_raw=False, whole_line=False,
                                         offset_key=None, src_pos=0, time=0, time_ns=None, tail=b"", out_cap=None):
        """split_regex_filter_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_split_regex_filter_parse_sls_lz4).  Returns (block, raw_len, number of pieces, counters[4])."""
        data, raw, nev, ctr, _m = self._split_regex(
            lib().lc_split_regex_filter_parse_sls_lz4, rx, buf, [split_char], keys, source_key, renamed_key,
            keep_fail, keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, False, tail,
            filt)
        return data, raw, nev, ctr

    def multiline_split_regex_filter_parse_sls(self, rx, buf, start, cont, end, discard, keys, source_key, filt,
                                               renamed_key=None, keep_fail=False, keep_succeed=False, copy_raw=False,
                                               whole_line=False, offset_key=None, src_pos=0, time=0, time_ns=None,
                                               out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_regex_filter_parse_sls).  Returns (bytes, number
        of events, counters[4], splitter counters[3])."""
        data, _raw, nev, ctr, mctr = self._split_regex(
            lib().lc_multiline_split_regex_filter_parse_sls, rx, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], keys, source_key, renamed_key, keep_fail,
            keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, True, None, filt)
        return data, nev, ctr, mctr

    def multiline_split_regex_filter_parse_sls_lz4(self, rx, buf, start, cont, end, discard, keys, source_key, filt,
                                                   renamed_key=None, keep_fail=False, keep_succeed=False,
                                                   copy_raw=False, whole_line=False, offset_key=None, src_pos=0,
                                                   time=0, time_ns=None, tail=b"", out_cap=None):
        """multiline_split_regex_filter_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_regex_filter_parse_sls_lz4).  Returns (block, raw_len, number of events, counters[4],
        splitter counters[3])."""
        return self._split_regex(
            lib().lc_multiline_split_regex_filter_parse_sls_lz4, rx, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], keys, source_key, renamed_key, keep_fail,
            keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, True, tail, filt)

    @staticmethod
    def _ts_args(tkey, ts, now, discard_interval, enable_ns):
        """the timestamp stage of the split -> regex -> timestamp calls: SourceKey tkey (bytes), the compiled
        Timestamp ts, now (time(NULL)), discard_interval (-1 = no history discard), enable_ns"""
        return [tkey, len(tkey), ts._h, int(now), int(discard_interval), int(bool(enable_ns))]

    def split_regex_timestamp_tap_dev(self, d_src, src_len, d_off, d_len, n, d_status, d_cap_off, d_cap_len,
                                      row_pitch, keys, source_key, tkey, d_val_off, d_val_len, renamed_key=None,
                                      keep_fail=False, keep_succeed=False, copy_raw=False, whole_line=False,
                                      offset_key=None):
        """The timestamp stage's value table (d_val_off, d_val_len; LC_TS_NO_KEY = no value) from the device piece
        and regex tables of the split -> regex chain (lc_split_regex_timestamp_tap_dev); queued, not waited for."""
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        _check(lib().lc_split_regex_timestamp_tap_dev(
            self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_cap_off), _p(d_cap_len),
            row_pitch, *cfg, int(bool(whole_line)), *self._sr_tail(offset_key, 0, 0, None)[:2], tkey, len(tkey),
            _p(d_val_off), _p(d_val_len)))

    def sls_serialize_split_regex_timestamp_dev(self, d_src, src_len, d_off, d_len, n, d_status, d_cap_off,
                                                d_cap_len, row_pitch, keys, source_key, d_ts_status, d_ts_sec,
                                                d_ts_nsec, enable_ns=False, renamed_key=None, keep_fail=False,
                                                keep_succeed=False, copy_raw=False, whole_line=False, offset_key=None,
                                                src_pos=0, time=0, time_ns=None, d_out=None, out_cap=0):
        """sls_serialize_split_regex_dev with each record's time from the device results of timestamp_parse_dev over
        the tap's value table (lc_sls_serialize_split_regex_timestamp_dev).  Returns (byte count, counters[8] = the
        regex stage's three, then key_not_found, out_failed, history_failure, discarded, out_successful); with d_out
        None the byte count needed."""
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        need = C.c_uint64(0)
        ctr = np.zeros(8, np.uint64)
        rc = lib().lc_sls_serialize_split_regex_timestamp_dev(
            self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_cap_off), _p(d_cap_len),
            row_pitch, *cfg, int(bool(whole_line)), *self._sr_tail(offset_key, src_pos, time, time_ns),
            _p(d_ts_status), _p(d_ts_sec), _p(d_ts_nsec), int(bool(enable_ns)), _p(d_out), out_cap, C.byref(need),
            _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def split_regex_timestamp_parse_sls(self, rx, buf, split_char, keys, source_key, tkey, ts, now,
                                        discard_interval=-1, enable_ns=False, renamed_key=None, keep_fail=False,
                                        keep_succeed=False, copy_raw=False, whole_line=False, offset_key=None,
                                        src_pos=0, time=0, time_ns=None, out_cap=None):
        """split_regex_parse_sls with ProcessorParseTimestampNative (SourceKey tkey, the compiled Timestamp ts)
        behind the regex stage (lc_split_regex_timestamp_parse_sls).  Returns (bytes, number of pieces,
        counters[8])."""
        data, _raw, nev, ctr, _m = self._split_regex(
            lib().lc_split_regex_timestamp_parse_sls, rx, buf, [split_char], keys, source_key, renamed_key,
            keep_fail, keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, False, None,
            None, self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, nev, ctr

    def split_regex_timestamp_parse_sls_lz4(self, rx, buf, split_char, keys, source_key, tkey, ts, now,
                                            discard_interval=-1, enable_ns=False, renamed_key=None, keep_fail=False,
                                            keep_succeed=False, copy_raw=False, whole_line=False, offset_key=None,
                                            src_pos=0, time=0, time_ns=None, tail=b"", out_cap=None):
        """split_regex_timestamp_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_split_regex_timestamp_parse_sls_lz4).  Returns (block, raw_len, number of pieces, counters[8])."""
        data, raw, nev, ctr, _m = self._split_regex(
            lib().lc_split_regex_timestamp_parse_sls_lz4, rx, buf, [split_char], keys, source_key, renamed_key,
            keep_fail, keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, False, tail,
            None, self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, raw, nev, ctr

    def multiline_split_regex_timestamp_parse_sls(self, rx, buf, start, cont, end, discard, keys, source_key, tkey,
                                                  ts, now, discard_interval=-1, enable_ns=False, renamed_key=None,
                                                  keep_fail=False, keep_succeed=False, copy_raw=False,
                                                  whole_line=False, offset_key=None, src_pos=0, time=0, time_ns=None,
                                                  out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_regex_timestamp_parse_sls).  Returns (bytes,
        number of events, counters[8], splitter counters[3])."""
        data, _raw, nev, ctr, mctr = self._split_regex(
            lib().lc_multiline_split_regex_timestamp_parse_sls, rx, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], keys, source_key, renamed_key, keep_fail,
            keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, True, None, None,
            self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, nev, ctr, mctr

    def multiline_split_regex_timestamp_parse_sls_lz4(self, rx, buf, start, cont, end, discard, keys, source_key,
                                                      tkey, ts, now, discard_interval=-1, enable_ns=False,
                                                      renamed_key=None, keep_fail=False, keep_succeed=False,
                                                      copy_raw=False, whole_line=False, offset_key=None, src_pos=0,
                                                      time=0, time_ns=None, tail=b"", out_cap=None):
        """multiline_split_regex_timestamp_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_regex_timestamp_parse_sls_lz4).  Returns (block, raw_len, number of events, counters[8],
        splitter counters[3])."""
        return self._split_regex(
            lib().lc_multiline_split_regex_timestamp_parse_sls_lz4, rx, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], keys, source_key, renamed_key, keep_fail,
            keep_succeed, copy_raw, whole_line, offset_key, src_pos, time, time_ns, out_cap, True, tail, None,
            self._ts_args(tkey, ts, now, discard_interval, enable_ns))

    def sls_serialize_split_delim_dev(self, d_src, src_len, d_off, d_len, n, d_status, d_nf, d_fo, d_fl, d_fd,
                                      max_fields, sep: bytes, quote, treatment, keys, source_key, renamed_key=None,
                                      keep_fail=False, keep_succeed=False, copy_raw=False, offset_key=None, src_pos=0,
                                      time=0, time_ns=None, d_out=None, out_cap=0):
        """Wire bytes of the split -> delimiter chain from the device piece tables of one split_lines_dev /
        multiline_split_dev call and the device tables of delim_parse_dev over those pieces (treatment: "extend" /
        "keep" / "discard"; lc_sls_serialize_split_delim_dev).  Returns (byte count written to d_out, counters[4] =
        successful, failed, discarded, blank); with d_out None the byte count needed."""
        sp = np.frombuffer(sep, np.uint8)
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        need = C.c_uint64(0)
        ctr = np.zeros(4, np.uint64)
        rc = lib().lc_sls_serialize_split_delim_dev(self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n,
                                                    _p(d_status), _p(d_nf), _p(d_fo), _p(d_fl), _p(d_fd), max_fields,
                                                    _p(sp), len(sep), quote, int(treatment == "extend"),
                                                    int(treatment == "discard"), *cfg,
                                                    *self._sr_tail(offset_key, src_pos, time, time_ns), _p(d_out),
                                                    out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def _split_delim(self, fn, buf, extra, sep, quote, treatment, keys, source_key, renamed_key, keep_fail,
                     keep_succeed, copy_raw, allow_short, max_fields, offset_key, src_pos, time, time_ns, out_cap, ml,
                     tail, ts_args=None):
        """one host-buffer split -> delimiter call, sized by an estimate first and by the exact size when that was
        short; tail None: the wire bytes, else records ‖ tail as one LZ4 block; ts_args: the timestamp stage of the
        split -> delimiter -> timestamp calls (_ts_args).  Returns (bytes, raw_len, n_events, counters[4], or [9] with
        ts_args, ml_counters[3] or None)"""
        a = _u8(buf)
        sp = np.frombuffer(sep, np.uint8)
        mf = int(max_fields if max_fields is not None else len(keys) + 16)
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        dcfg = [_p(sp), len(sep), quote, int(treatment == "extend"), int(treatment == "discard"),
                int(bool(allow_short)), mf]
        tl = None if tail is None else np.frombuffer(bytes(tail), np.uint8)
        est = 2 * a.size + 4096 + (0 if tl is None else tl.size)
        cap = int(out_cap if out_cap is not None else est + est // 255 + 16)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
            ctr, mctr = np.zeros(9 if ts_args else 4, np.uint64), np.zeros(3, np.uint64)
            z = [] if tl is None else [_p(tl) if tl.size else None, tl.size]
            outs = [_p(out), cap, C.byref(need)] + ([] if tl is None else [C.byref(raw)]) + [C.byref(nev), _p(ctr)]
            rc = fn(self._h, _p(a), a.size, *extra, *dcfg, *cfg, *self._sr_tail(offset_key, src_pos, time, time_ns),
                    *(ts_args or []), *z, *outs, *([_p(mctr)] if ml else []))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), int(raw.value), int(nev.value), ctr, (mctr if ml else None)
        _check(rc)

    def split_delim_parse_sls(self, buf, split_char, sep: bytes, quote, treatment, keys, source_key, renamed_key=None,
                              keep_fail=False, keep_succeed=False, copy_raw=False, allow_short=True, max_fields=None,
                              offset_key=None, src_pos=0, time=0, time_ns=None, out_cap=None):
        """Host source value in: split, delimiter, wire bytes out (lc_split_delim_parse_sls).  Returns (bytes, number
        of pieces, counters[4] = successful, failed, discarded, blank)."""
        data, _raw, nev, ctr, _m = self._split_delim(
            lib().lc_split_delim_parse_sls, buf, [split_char], sep, quote, treatment, keys, source_key, renamed_key,
            keep_fail, keep_succeed, copy_raw, allow_short, max_fields, offset_key, src_pos, time, time_ns, out_cap,
            False, None)
        return data, nev, ctr

    def split_delim_parse_sls_lz4(self, buf, split_char, sep: bytes, quote, treatment, keys, source_key,
                                  renamed_key=None, keep_fail=False, keep_succeed=False, copy_raw=False,
                                  allow_short=True, max_fields=None, offset_key=None, src_pos=0, time=0, time_ns=None,
                                  tail=b"", out_cap=None):
        """split_delim_parse_sls's records followed by `tail` as ONE LZ4 block (lc_split_delim_parse_sls_lz4).
        Returns (block, raw_len, number of pieces, counters[4])."""
        data, raw, nev, ctr, _m = self._split_delim(
            lib().lc_split_delim_parse_sls_lz4, buf, [split_char], sep, quote, treatment, keys, source_key,
            renamed_key, keep_fail, keep_succeed, copy_raw, allow_short, max_fields, offset_key, src_pos, time,
            time_ns, out_cap, False, tail)
        return data, raw, nev, ctr

    def multiline_split_delim_parse_sls(self, buf, start, cont, end, discard, sep: bytes, quote, treatment, keys,
                                        source_key, renamed_key=None, keep_fail=False, keep_succeed=False,
                                        copy_raw=False, allow_short=True, max_fields=None, offset_key=None, src_pos=0,
                                        time=0, time_ns=None, out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_delim_parse_sls).  Returns (bytes, number of
        events, counters[4], splitter counters[3] = matched_events, input_lines, unmatched_lines)."""
        data, _raw, nev, ctr, mctr = self._split_delim(
            lib().lc_multiline_split_delim_parse_sls, buf, [_rh(start), _rh(cont), _rh(end), int(bool(discard))], sep,
            quote, treatment, keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw, allow_short,
            max_fields, offset_key, src_pos, time, time_ns, out_cap, True, None)
        return data, nev, ctr, mctr

    def multiline_split_delim_parse_sls_lz4(self, buf, start, cont, end, discard, sep: bytes, quote, treatment, keys,
                                            source_key, renamed_key=None, keep_fail=False, keep_succeed=False,
                                            copy_raw=False, allow_short=True, max_fields=None, offset_key=None,
                                            src_pos=0, time=0, time_ns=None, tail=b"", out_cap=None):
        """multiline_split_delim_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_delim_parse_sls_lz4).  Returns (block, raw_len, number of events, counters[4], splitter
        counters[3])."""
        return self._split_delim(
            lib().lc_multiline_split_delim_parse_sls_lz4, buf, [_rh(start), _rh(cont), _rh(end), int(bool(discard))],
            sep, quote, treatment, keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw, allow_short,
            max_fields, offset_key, src_pos, time, time_ns, out_cap, True, tail)

    def split_delim_timestamp_tap_dev(self, d_src, src_len, d_off, d_len, n, d_status, d_nf, d_fo, d_fl, d_fd,
                                      max_fields, sep: bytes, quote, treatment, keys, source_key, tkey, d_val, val_cap,
                                      d_val_off, d_val_len, renamed_key=None, keep_fail=False, keep_succeed=False,
                                      copy_raw=False, offset_key=None):
        """The timestamp stage's value table (d_val_off, d_val_len; LC_TS_NO_KEY = no value) over d_val, with each
        value copied into d_val (val_cap >= src_len) at its own offset, from the device piece and delimiter tables of
        the split -> delimiter chain (lc_split_delim_timestamp_tap_dev); queued, not waited for."""
        sp = np.frombuffer(sep, np.uint8)
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        _check(lib().lc_split_delim_timestamp_tap_dev(
            self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_nf), _p(d_fo), _p(d_fl),
            _p(d_fd), max_fields, _p(sp), len(sep), quote, int(treatment == "extend"), int(treatment == "discard"),
            *cfg, *self._sr_tail(offset_key, 0, 0, None)[:2], tkey, len(tkey), _p(d_val), val_cap, _p(d_val_off),
            _p(d_val_len)))

    def sls_serialize_split_delim_timestamp_dev(self, d_src, src_len, d_off, d_len, n, d_status, d_nf, d_fo, d_fl,
                                                d_fd, max_fields, sep: bytes, quote, treatment, keys, source_key,
                                                d_ts_status, d_ts_sec, d_ts_nsec, enable_ns=False, renamed_key=None,
                                                keep_fail=False, keep_succeed=False, copy_raw=False, offset_key=None,
                                                src_pos=0, time=0, time_ns=None, d_out=None, out_cap=0):
        """sls_serialize_split_delim_dev with each record's time from the device results of timestamp_parse_dev over
        the tap's value table (lc_sls_serialize_split_delim_timestamp_dev).  Returns (byte count, counters[9] = the
        delimiter stage's four, then key_not_found, out_failed, history_failure, discarded, out_successful); with
        d_out None the byte count needed."""
        sp = np.frombuffer(sep, np.uint8)
        _keep, cfg = self._delim_sls_cfg(keys, source_key, renamed_key, keep_fail, keep_succeed, copy_raw)
        need = C.c_uint64(0)
        ctr = np.zeros(9, np.uint64)
        rc = lib().lc_sls_serialize_split_delim_timestamp_dev(
            self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_nf), _p(d_fo), _p(d_fl),
            _p(d_fd), max_fields, _p(sp), len(sep), quote, int(treatment == "extend"), int(treatment == "discard"),
            *cfg, *self._sr_tail(offset_key, src_pos, time, time_ns), _p(d_ts_status), _p(d_ts_sec), _p(d_ts_nsec),
            int(bool(enable_ns)), _p(d_out), out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def split_delim_timestamp_parse_sls(self, buf, split_char, sep: bytes, quote, treatment, keys, source_key, tkey,
                                        ts, now, discard_interval=-1, enable_ns=False, renamed_key=None,
                                        keep_fail=False, keep_succeed=False, copy_raw=False, allow_short=True,
                                        max_fields=None, offset_key=None, src_pos=0, time=0, time_ns=None,
                                        out_cap=None):
        """split_delim_parse_sls with ProcessorParseTimestampNative (SourceKey tkey, the compiled Timestamp ts) behind
        the delimiter stage (lc_split_delim_timestamp_parse_sls).  Returns (bytes, number of pieces, counters[9])."""
        data, _raw, nev, ctr, _m = self._split_delim(
            lib().lc_split_delim_timestamp_parse_sls, buf, [split_char], sep, quote, treatment, keys, source_key,
            renamed_key, keep_fail, keep_succeed, copy_raw, allow_short, max_fields, offset_key, src_pos, time,
            time_ns, out_cap, False, None, self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, nev, ctr

    def split_delim_timestamp_parse_sls_lz4(self, buf, split_char, sep: bytes, quote, treatment, keys, source_key,
                                            tkey, ts, now, discard_interval=-1, enable_ns=False, renamed_key=None,
                                            keep_fail=False, keep_succeed=False, copy_raw=False, allow_short=True,
                                            max_fields=None, offset_key=None, src_pos=0, time=0, time_ns=None,
                                            tail=b"", out_cap=None):
        """split_delim_timestamp_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_split_delim_timestamp_parse_sls_lz4).  Returns (block, raw_len, number of pieces, counters[9])."""
        data, raw, nev, ctr, _m = self._split_delim(
            lib().lc_split_delim_timestamp_parse_sls_lz4, buf, [split_char], sep, quote, treatment, keys, source_key,
            renamed_key, keep_fail, keep_succeed, copy_raw, allow_short, max_fields, offset_key, src_pos, time,
            time_ns, out_cap, False, tail, self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, raw, nev, ctr

    def multiline_split_delim_timestamp_parse_sls(self, buf, start, cont, end, discard, sep: bytes, quote, treatment,
                                                  keys, source_key, tkey, ts, now, discard_interval=-1,
                                                  enable_ns=False, renamed_key=None, keep_fail=False,
                                                  keep_succeed=False, copy_raw=False, allow_short=True,
                                                  max_fields=None, offset_key=None, src_pos=0, time=0, time_ns=None,
                                                  out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_delim_timestamp_parse_sls).  Returns (bytes,
        number of events, counters[9], splitter counters[3])."""
        data, _raw, nev, ctr, mctr = self._split_delim(
            lib().lc_multiline_split_delim_timestamp_parse_sls, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], sep, quote, treatment, keys, source_key,
            renamed_key, keep_fail, keep_succeed, copy_raw, allow_short, max_fields, offset_key, src_pos, time,
            time_ns, out_cap, True, None, self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, nev, ctr, mctr

    def multiline_split_delim_timestamp_parse_sls_lz4(self, buf, start, cont, end, discard, sep: bytes, quote,
                                                      treatment, keys, source_key, tkey, ts, now, discard_interval=-1,
                                                      enable_ns=False, renamed_key=None, keep_fail=False,
                                                      keep_succeed=False, copy_raw=False, allow_short=True,
                                                      max_fields=None, offset_key=None, src_pos=0, time=0,
                                                      time_ns=None, tail=b"", out_cap=None):
        """multiline_split_delim_timestamp_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_delim_timestamp_parse_sls_lz4).  Returns (block, raw_len, number of events,
        counters[9], splitter counters[3])."""
        return self._split_delim(
            lib().lc_multiline_split_delim_timestamp_parse_sls_lz4, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], sep, quote, treatment, keys, source_key,
            renamed_key, keep_fail, keep_succeed, copy_raw, allow_short, max_fields, offset_key, src_pos, time,
            time_ns, out_cap, True, tail, self._ts_args(tkey, ts, now, discard_interval, enable_ns))

    def sls_serialize_split_delim_regex_dev(self, d_src, src_len, d_off, d_len, n, d_status, d_nf, d_fo, d_fl, d_fd,
                                            max_fields, delim, regex, d_val_off, d_val_len, d_re_status, d_cap_off,
                                            d_cap_len, row_pitch, offset_key=None, src_pos=0, time=0, time_ns=None,
                                            d_out=None, out_cap=0):
        """Wire bytes of the split -> delimiter -> regex chain from the device piece tables of one split_lines_dev /
        multiline_split_dev call, the device tables of delim_parse_dev over those pieces, the value table of
        delim_regex_tap_dev over the same tables and the regex tables over the values (delim, regex: as for
        sls_serialize_delim_regex_dev; lc_sls_serialize_split_delim_regex_dev).  Returns (byte count written to d_out,
        counters[8]); with d_out None the byte count needed."""
        _keep, cfg = self._chain_cfg(delim, regex)
        need = C.c_uint64(0)
        ctr = np.zeros(8, np.uint64)
        rc = lib().lc_sls_serialize_split_delim_regex_dev(
            self._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_nf), _p(d_fo), _p(d_fl),
            _p(d_fd), max_fields, *cfg, *self._sr_tail(offset_key, src_pos, time, time_ns), _p(d_val_off),
            _p(d_val_len), _p(d_re_status), _p(d_cap_off), _p(d_cap_len), row_pitch, _p(d_out), out_cap,
            C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def _split_delim_regex(self, fn, rx, buf, extra, delim, regex, allow_short, max_fields, offset_key, src_pos, time,
                           time_ns, out_cap, ml, tail):
        """one host-buffer split -> delimiter -> regex call, sized by an estimate first and by the exact size when that
        was short; tail None: the wire bytes, else records ‖ tail as one LZ4 block.  Returns (bytes, raw_len,
        n_events, counters[8], ml_counters[3] or None)"""
        a = _u8(buf)
        mf = int(max_fields if max_fields is not None else len(delim["keys"]) + 16)
        _keep, cfg = self._chain_cfg(delim, regex)
        tl = None if tail is None else np.frombuffer(bytes(tail), np.uint8)
        est = 2 * a.size + 4096 + (0 if tl is None else tl.size)
        cap = int(out_cap if out_cap is not None else est + est // 255 + 16)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
            ctr, mctr = np.zeros(8, np.uint64), np.zeros(3, np.uint64)
            z = [] if tl is None else [_p(tl) if tl.size else None, tl.size]
            outs = [_p(out), cap, C.byref(need)] + ([] if tl is None else [C.byref(raw)]) + [C.byref(nev), _p(ctr)]
            rc = fn(self._h, _rh(rx), _p(a), a.size, *extra, int(bool(allow_short)), mf, *cfg,
                    *self._sr_tail(offset_key, src_pos, time, time_ns), *z, *outs, *([_p(mctr)] if ml else []))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), int(raw.value), int(nev.value), ctr, (mctr if ml else None)
        _check(rc)

    def split_delim_regex_parse_sls(self, rx, buf, split_char, delim, regex, allow_short=True, max_fields=None,
                                    offset_key=None, src_pos=0, time=0, time_ns=None, out_cap=None):
        """Host source value in: split, delimiter, regex on one of its keys, wire bytes out
        (lc_split_delim_regex_parse_sls; rx may be None in whole-line mode; delim, regex as for
        sls_serialize_delim_regex_dev).  Returns (bytes, number of pieces, counters[8])."""
        data, _raw, nev, ctr, _m = self._split_delim_regex(
            lib().lc_split_delim_regex_parse_sls, rx, buf, [split_char], delim, regex, allow_short, max_fields,
            offset_key, src_pos, time, time_ns, out_cap, False, None)
        return data, nev, ctr

    def split_delim_regex_parse_sls_lz4(self, rx, buf, split_char, delim, regex, allow_short=True, max_fields=None,
                                        offset_key=None, src_pos=0, time=0, time_ns=None, tail=b"", out_cap=None):
        """split_delim_regex_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_split_delim_regex_parse_sls_lz4).  Returns (block, raw_len, number of pieces, counters[8])."""
        data, raw, nev, ctr, _m = self._split_delim_regex(
            lib().lc_split_delim_regex_parse_sls_lz4, rx, buf, [split_char], delim, regex, allow_short, max_fields,
            offset_key, src_pos, time, time_ns, out_cap, False, tail)
        return data, raw, nev, ctr

    def multiline_split_delim_regex_parse_sls(self, rx, buf, start, cont, end, discard, delim, regex,
                                              allow_short=True, max_fields=None, offset_key=None, src_pos=0, time=0,
                                              time_ns=None, out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_delim_regex_parse_sls).  Returns (bytes, number
        of events, counters[8], splitter counters[3] = matched_events, input_lines, unmatched_lines)."""
        data, _raw, nev, ctr, mctr = self._split_delim_regex(
            lib().lc_multiline_split_delim_regex_parse_sls, rx, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], delim, regex, allow_short, max_fields, offset_key,
            src_pos, time, time_ns, out_cap, True, None)
        return data, nev, ctr, mctr

    def multiline_split_delim_regex_parse_sls_lz4(self, rx, buf, start, cont, end, discard, delim, regex,
                                                  allow_short=True, max_fields=None, offset_key=None, src_pos=0,
                                                  time=0, time_ns=None, tail=b"", out_cap=None):
        """multiline_split_delim_regex_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_delim_regex_parse_sls_lz4).  Returns (block, raw_len, number of events, counters[8],
        splitter counters[3])."""
        return self._split_delim_regex(
            lib().lc_multiline_split_delim_regex_parse_sls_lz4, rx, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], delim, regex, allow_short, max_fields, offset_key,
            src_pos, time, time_ns, out_cap, True, tail)

    def lz4_compress_dev(self, d_in, nseg, d_seg_off, d_seg_len, d_out=None, out_cap=0, d_blk_off=None,
                         d_blk_len=None):
        """One LZ4 block per device segment d_in[d_seg_off[g], + d_seg_len[g]) (u64 / u32 tables), packed in d_out
        with the table d_blk_off (u64) / d_blk_len (u32) (lc_lz4_compress_dev).  Returns the byte count written to
        d_out, or with d_out None the byte count needed."""
        need = C.c_uint64(0)
        rc = lib().lc_lz4_compress_dev(self._h, _p(d_in), nseg, _p(d_seg_off), _p(d_seg_len), _p(d_out), out_cap,
                                       _p(d_blk_off), _p(d_blk_len), C.byref(need))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value)  # a sizing query
        _check(rc)
        return int(need.value)

    def lz4_compress(self, segments, out_cap=None):
        """Host segments (bytes-like) in, one LZ4 block each out (lc_lz4_compress).  Returns the list of blocks."""
        segs = [_u8(s) for s in segments]
        n = len(segs)
        ptrs = (C.c_void_p * max(n, 1))(*[s.ctypes.data for s in segs])
        lens = np.array([s.size for s in segs] or [0], np.uint32)
        cap = int(out_cap if out_cap is not None else sum(int(x) + int(x) // 255 + 16 for x in lens))
        out = np.empty(max(cap, 1), np.uint8)
        boff, blen = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint32)
        need = C.c_uint64(0)
        _check(lib().lc_lz4_compress(self._h, n, C.cast(ptrs, C.c_void_p), _p(lens), _p(out), cap, _p(boff),
                                     _p(blen), C.byref(need)))
        return [bytes(out[int(o):int(o) + int(ln)]) for o, ln in zip(boff[:n], blen[:n])]

    def zstd_compress_dev(self, d_in, nseg, d_seg_off, d_seg_len, d_out=None, out_cap=0, d_frm_off=None,
                          d_frm_len=None):
        """One zstd frame per device segment d_in[d_seg_off[g], + d_seg_len[g]) (u64 / u32 tables), packed in d_out
        with the table d_frm_off (u64) / d_frm_len (u32) (lc_zstd_compress_dev).  Returns the byte count written to
        d_out, or with d_out None the byte count needed."""
        need = C.c_uint64(0)
        rc = lib().lc_zstd_compress_dev(self._h, _p(d_in), nseg, _p(d_seg_off), _p(d_seg_len), _p(d_out), out_cap,
                                        _p(d_frm_off), _p(d_frm_len), C.byref(need))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value)  # a sizing query
        _check(rc)
        return int(need.value)

    def zstd_compress(self, segments, out_cap=None):
        """Host segments (bytes-like) in, one zstd frame each out (lc_zstd_compress).  Returns the list of frames."""
        segs = [_u8(s) for s in segments]
        n = len(segs)
        ptrs = (C.c_void_p * max(n, 1))(*[s.ctypes.data for s in segs])
        lens = np.array([s.size for s in segs] or [0], np.uint32)
        cap = int(out_cap if out_cap is not None else sum(zstd_bound(int(x)) for x in lens[:n]))
        out = np.empty(max(cap, 1), np.uint8)
        foff, flen = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint32)
        need = C.c_uint64(0)
        _check(lib().lc_zstd_compress(self._h, n, C.cast(ptrs, C.c_void_p), _p(lens), _p(out), cap, _p(foff),
                                      _p(flen), C.byref(need)))
        return [bytes(out[int(o):int(o) + int(ln)]) for o, ln in zip(foff[:n], flen[:n])]

    def split_lines_dev(self, d_buf, length, split_char, d_off, d_len, cap):
        n = C.c_uint64(0)
        _check(lib().lc_split_lines_dev(self._h, _p(d_buf), length, split_char, _p(d_off), _p(d_len), cap,
                                        C.byref(n)))
        return n.value

    def timestamp_parse(self, ts, base, ev_off, ev_len, grp, now, discard_interval=43200):
        """ProcessorParseTimestampNative over host buffers (lc_timestamp_parse): ev_len LC_TS_NO_KEY = no SourceKey,
        grp = group starts plus n.  Returns (status u8, sec i64, nsec u32, counters u64[5])."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        grp = np.ascontiguousarray(grp, np.uint32)
        n = ev_off.size
        st, sec, ns = np.empty(n, np.uint8), np.empty(n, np.int64), np.empty(n, np.uint32)
        cnt = np.zeros(5, np.uint64)
        _check(lib().lc_timestamp_parse(self._h, ts._h, _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(grp),
                                        max(grp.size - 1, 0), int(now), int(discard_interval), _p(sec), _p(ns),
                                        _p(st), _p(cnt)))
        return st, sec, ns, cnt

    def apsara_parse(self, ap, base, ev_off, ev_len, grp, now, discard_interval=43200, entry_cap=None):
        """ProcessorParseApsaraNative over host buffers (lc_apsara_parse): ev_len LC_TS_NO_KEY = no SourceKey, grp =
        group starts plus n.  entry_cap None sizes the entries with a first call.  Returns (status u8, sec i64,
        nsec u32, micro i64, first u64[n + 1], entries u32[m, 4], counters u64[5])."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        grp = np.ascontiguousarray(grp, np.uint32)
        n = ev_off.size
        st, sec, ns = np.empty(n, np.uint8), np.empty(n, np.int64), np.empty(n, np.uint32)
        us, first = np.empty(n, np.int64), np.empty(n + 1, np.uint64)
        cnt = np.zeros(5, np.uint64)
        m = C.c_uint64(0)

        def call(cap, ent):
            return lib().lc_apsara_parse(self._h, ap._h, _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(grp),
                                         max(grp.size - 1, 0), int(now), int(discard_interval), _p(st), _p(sec),
                                         _p(ns), _p(us), _p(first), _p(ent), cap, C.byref(m), _p(cnt))
        if entry_cap is None:
            rc = call(0, np.zeros((1, 4), np.uint32))
            if rc not in (LC_OK, LC_ERR_CAPACITY):
                _check(rc)
            entry_cap = m.value
        ent = np.zeros((max(int(entry_cap), 1), 4), np.uint32)
        _check(call(int(entry_cap), ent))
        return st, sec, ns, us, first, ent[:m.value], cnt

    def apsara_parse_dev(self, ap, d_base, base_len, d_ev_off, d_ev_len, n, d_grp, ngroups, now, discard_interval,
                         d_status, d_sec, d_nsec, d_micro, d_first, d_entries, entry_cap, d_counters):
        """lc_apsara_parse_dev over device tables; waits for the device.  Returns the entry count (raises LcError
        with LC_ERR_CAPACITY when it exceeds entry_cap; no entry is written then)."""
        m = C.c_uint64(0)
        _check(lib().lc_apsara_parse_dev(self._h, ap._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len), n,
                                         _p(d_grp), ngroups, int(now), int(discard_interval), _p(d_status), _p(d_sec),
                                         _p(d_nsec), _p(d_micro), _p(d_first), _p(d_entries), entry_cap, C.byref(m),
                                         _p(d_counters)))
        return m.value

    def json_parse(self, js, base, ev_off, ev_len, entry_cap=None, arena_cap=None):
        """ProcessorParseJsonNative over host buffers (lc_json_parse): ev_len LC_TS_NO_KEY = no SourceKey.  Caps of
        None size the outputs with a first call.  Returns (status u8, first u64[n + 1], entries u32[m, 4], arena bytes,
        counters u64[3])."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        n = ev_off.size
        st, first, cnt = np.empty(n, np.uint8), np.empty(n + 1, np.uint64), np.zeros(3, np.uint64)
        m, ab = C.c_uint64(0), C.c_uint64(0)

        def call(ecap, ent, acap, ar):
            return lib().lc_json_parse(self._h, js._h, _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(st), _p(first),
                                       _p(ent), ecap, C.byref(m), _p(ar), acap, C.byref(ab), _p(cnt))
        if entry_cap is None or arena_cap is None:
            rc = call(0, np.zeros((1, 4), np.uint32), 0, np.zeros(1, np.uint8))
            if rc not in (LC_OK, LC_ERR_CAPACITY):
                _check(rc)
            entry_cap = m.value if entry_cap is None else entry_cap
            arena_cap = ab.value if arena_cap is None else arena_cap
        ent = np.zeros((max(int(entry_cap), 1), 4), np.uint32)
        ar = np.zeros(max(int(arena_cap), 1), np.uint8)
        _check(call(int(entry_cap), ent, int(arena_cap), ar))
        return st, first, ent[:m.value], ar[:ab.value].tobytes(), cnt

    def _sj_cfg(self, renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns):
        r = renamed_key or b""
        return [r, len(r), int(bool(keep_fail)), int(bool(keep_succeed)), int(bool(copy_raw))] + \
            self._sr_tail(offset_key, src_pos, time, time_ns)

    def sls_serialize_split_json_dev(self, js, d_src, src_len, d_off, d_len, n, d_status, d_first, d_entries, d_arena,
                                     renamed_key, keep_fail=False, keep_succeed=False, copy_raw=False,
                                     offset_key=None, src_pos=0, time=0, time_ns=None, d_out=None, out_cap=0):
        """Wire bytes of the split -> JSON chain from the device piece tables of one split_lines_dev /
        multiline_split_dev call and the device tables of json_parse_dev over those pieces with js
        (lc_sls_serialize_split_json_dev); renamed_key is the effective RenamedSourceKey.  Returns (byte count
        written to d_out, counters[3] = successful, failed, discarded); with d_out None the byte count needed."""
        need = C.c_uint64(0)
        ctr = np.zeros(3, np.uint64)
        rc = lib().lc_sls_serialize_split_json_dev(
            self._h, js._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_first), _p(d_entries),
            _p(d_arena), *self._sj_cfg(renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time,
                                       time_ns), _p(d_out), out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def _split_json(self, fn, js, buf, extra, renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos,
                    time, time_ns, out_cap, ml, tail, ts_args=None):
        """one host-buffer split -> JSON call, sized by an estimate first and by the exact size when that was short;
        tail None: the wire bytes, else records ‖ tail as one LZ4 block; ts_args: the timestamp stage of the
        split -> JSON -> timestamp calls (_ts_args).  Returns (bytes, raw_len, n_events, counters[3], or [8] with
        ts_args, ml_counters[3] or None)"""
        a = _u8(buf)
        cfg = self._sj_cfg(renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns) + \
            (ts_args or [])
        tl = None if tail is None else np.frombuffer(bytes(tail), np.uint8)
        est = 2 * a.size + 4096 + (0 if tl is None else tl.size)
        cap = int(out_cap if out_cap is not None else est + est // 255 + 16)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
            ctr, mctr = np.zeros(8 if ts_args else 3, np.uint64), np.zeros(3, np.uint64)
            z = [] if tl is None else [_p(tl) if tl.size else None, tl.size]
            outs = [_p(out), cap, C.byref(need)] + ([] if tl is None else [C.byref(raw)]) + [C.byref(nev), _p(ctr)]
            rc = fn(self._h, js._h, _p(a), a.size, *extra, *cfg, *z, *outs, *([_p(mctr)] if ml else []))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), int(raw.value), int(nev.value), ctr, (mctr if ml else None)
        _check(rc)

    def split_json_parse_sls(self, js, buf, split_char, renamed_key, keep_fail=False, keep_succeed=False,
                             copy_raw=False, offset_key=None, src_pos=0, time=0, time_ns=None, out_cap=None):
        """Host source value in: split, JSON, wire bytes out (lc_split_json_parse_sls).  Returns (bytes, number of
        pieces, counters[3])."""
        data, _raw, nev, ctr, _m = self._split_json(
            lib().lc_split_json_parse_sls, js, buf, [split_char], renamed_key, keep_fail, keep_succeed, copy_raw,
            offset_key, src_pos, time, time_ns, out_cap, False, None)
        return data, nev, ctr

    def split_json_parse_sls_lz4(self, js, buf, split_char, renamed_key, keep_fail=False, keep_succeed=False,
                                 copy_raw=False, offset_key=None, src_pos=0, time=0, time_ns=None, tail=b"",
                                 out_cap=None):
        """split_json_parse_sls's records followed by `tail` as ONE LZ4 block (lc_split_json_parse_sls_lz4).
        Returns (block, raw_len, number of pieces, counters[3])."""
        data, raw, nev, ctr, _m = self._split_json(
            lib().lc_split_json_parse_sls_lz4, js, buf, [split_char], renamed_key, keep_fail, keep_succeed, copy_raw,
            offset_key, src_pos, time, time_ns, out_cap, False, tail)
        return data, raw, nev, ctr

    def multiline_split_json_parse_sls(self, js, buf, start, cont, end, discard, renamed_key, keep_fail=False,
                                       keep_succeed=False, copy_raw=False, offset_key=None, src_pos=0, time=0,
                                       time_ns=None, out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_json_parse_sls).  Returns (bytes, number of
        events, counters[3], splitter counters[3])."""
        data, _raw, nev, ctr, mctr = self._split_json(
            lib().lc_multiline_split_json_parse_sls, js, buf, [_rh(start), _rh(cont), _rh(end), int(bool(discard))],
            renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns, out_cap, True, None)
        return data, nev, ctr, mctr

    def multiline_split_json_parse_sls_lz4(self, js, buf, start, cont, end, discard, renamed_key, keep_fail=False,
                                           keep_succeed=False, copy_raw=False, offset_key=None, src_pos=0, time=0,
                                           time_ns=None, tail=b"", out_cap=None):
        """multiline_split_json_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_json_parse_sls_lz4).  Returns (block, raw_len, number of events, counters[3], splitter
        counters[3])."""
        return self._split_json(
            lib().lc_multiline_split_json_parse_sls_lz4, js, buf, [_rh(start), _rh(cont), _rh(end), int(bool(discard))],
            renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns, out_cap, True, tail)

    def split_json_timestamp_tap_dev(self, js, d_src, src_len, d_off, d_len, n, d_status, d_first, d_entries,
                                     d_arena, renamed_key, tkey, d_val, val_cap, d_val_off, d_val_len,
                                     keep_fail=False, keep_succeed=False, copy_raw=False, offset_key=None):
        """The timestamp stage's value table (d_val_off, d_val_len; LC_TS_NO_KEY = no value) over d_val, with each
        value copied into d_val (val_cap >= src_len + the arena's bytes), from the device piece and JSON tables of
        the split -> JSON chain (lc_split_json_timestamp_tap_dev); queued, not waited for."""
        r = renamed_key or b""
        _check(lib().lc_split_json_timestamp_tap_dev(
            self._h, js._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_first), _p(d_entries),
            _p(d_arena), r, len(r), int(bool(keep_fail)), int(bool(keep_succeed)), int(bool(copy_raw)),
            *self._sr_tail(offset_key, 0, 0, None)[:2], tkey, len(tkey), _p(d_val), val_cap, _p(d_val_off),
            _p(d_val_len)))

    def sls_serialize_split_json_timestamp_dev(self, js, d_src, src_len, d_off, d_len, n, d_status, d_first,
                                               d_entries, d_arena, renamed_key, d_ts_status, d_ts_sec, d_ts_nsec,
                                               enable_ns=False, keep_fail=False, keep_succeed=False, copy_raw=False,
                                               offset_key=None, src_pos=0, time=0, time_ns=None, d_out=None,
                                               out_cap=0):
        """sls_serialize_split_json_dev with each record's time from the device results of timestamp_parse_dev over
        the tap's value table (lc_sls_serialize_split_json_timestamp_dev).  Returns (byte count, counters[8] = the
        JSON stage's three, then key_not_found, out_failed, history_failure, discarded, out_successful); with d_out
        None the byte count needed."""
        need = C.c_uint64(0)
        ctr = np.zeros(8, np.uint64)
        rc = lib().lc_sls_serialize_split_json_timestamp_dev(
            self._h, js._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_first), _p(d_entries),
            _p(d_arena), *self._sj_cfg(renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time,
                                       time_ns), _p(d_ts_status), _p(d_ts_sec), _p(d_ts_nsec), int(bool(enable_ns)),
            _p(d_out), out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def split_json_timestamp_parse_sls(self, js, buf, split_char, renamed_key, tkey, ts, now, discard_interval=-1,
                                       enable_ns=False, keep_fail=False, keep_succeed=False, copy_raw=False,
                                       offset_key=None, src_pos=0, time=0, time_ns=None, out_cap=None):
        """split_json_parse_sls with ProcessorParseTimestampNative (SourceKey tkey, the compiled Timestamp ts) behind
        the JSON stage (lc_split_json_timestamp_parse_sls).  Returns (bytes, number of pieces, counters[8])."""
        data, _raw, nev, ctr, _m = self._split_json(
            lib().lc_split_json_timestamp_parse_sls, js, buf, [split_char], renamed_key, keep_fail, keep_succeed,
            copy_raw, offset_key, src_pos, time, time_ns, out_cap, False, None,
            self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, nev, ctr

    def split_json_timestamp_parse_sls_lz4(self, js, buf, split_char, renamed_key, tkey, ts, now,
                                           discard_interval=-1, enable_ns=False, keep_fail=False,
                                           keep_succeed=False, copy_raw=False, offset_key=None, src_pos=0, time=0,
                                           time_ns=None, tail=b"", out_cap=None):
        """split_json_timestamp_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_split_json_timestamp_parse_sls_lz4).  Returns (block, raw_len, number of pieces, counters[8])."""
        data, raw, nev, ctr, _m = self._split_json(
            lib().lc_split_json_timestamp_parse_sls_lz4, js, buf, [split_char], renamed_key, keep_fail, keep_succeed,
            copy_raw, offset_key, src_pos, time, time_ns, out_cap, False, tail,
            self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, raw, nev, ctr

    def multiline_split_json_timestamp_parse_sls(self, js, buf, start, cont, end, discard, renamed_key, tkey, ts, now,
                                                 discard_interval=-1, enable_ns=False, keep_fail=False,
                                                 keep_succeed=False, copy_raw=False, offset_key=None, src_pos=0,
                                                 time=0, time_ns=None, out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_json_timestamp_parse_sls).  Returns (bytes,
        number of events, counters[8], splitter counters[3])."""
        data, _raw, nev, ctr, mctr = self._split_json(
            lib().lc_multiline_split_json_timestamp_parse_sls, js, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], renamed_key, keep_fail, keep_succeed, copy_raw,
            offset_key, src_pos, time, time_ns, out_cap, True, None,
            self._ts_args(tkey, ts, now, discard_interval, enable_ns))
        return data, nev, ctr, mctr

    def multiline_split_json_timestamp_parse_sls_lz4(self, js, buf, start, cont, end, discard, renamed_key, tkey, ts,
                                                     now, discard_interval=-1, enable_ns=False, keep_fail=False,
                                                     keep_succeed=False, copy_raw=False, offset_key=None, src_pos=0,
                                                     time=0, time_ns=None, tail=b"", out_cap=None):
        """multiline_split_json_timestamp_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_json_timestamp_parse_sls_lz4).  Returns (block, raw_len, number of events,
        counters[8], splitter counters[3])."""
        return self._split_json(
            lib().lc_multiline_split_json_timestamp_parse_sls_lz4, js, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], renamed_key, keep_fail, keep_succeed, copy_raw,
            offset_key, src_pos, time, time_ns, out_cap, True, tail,
            self._ts_args(tkey, ts, now, discard_interval, enable_ns))

    def _sa_cfg(self, renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns, enable_ns):
        r = renamed_key or b""
        return [r, len(r), int(bool(keep_fail)), int(bool(keep_succeed)), int(bool(copy_raw))] + \
            self._sr_tail(offset_key, src_pos, time, time_ns) + [int(bool(enable_ns))]

    def sls_serialize_split_apsara_dev(self, ap, d_src, src_len, d_off, d_len, n, d_status, d_sec, d_nsec, d_micro,
                                       d_first, d_entries, renamed_key, keep_fail=False, keep_succeed=False,
                                       copy_raw=False, offset_key=None, src_pos=0, time=0, time_ns=None,
                                       enable_ns=False, d_out=None, out_cap=0):
        """Wire bytes of the split -> Apsara chain from the device piece tables of one split_lines_dev /
        multiline_split_dev call and the device tables of apsara_parse_dev over those pieces with ap, d_src as base and
        one group (lc_sls_serialize_split_apsara_dev); renamed_key is the effective RenamedSourceKey.  Returns (byte
        count written to d_out, counters[5] in lc_apsara_parse's order); with d_out None the byte count needed."""
        need = C.c_uint64(0)
        ctr = np.zeros(5, np.uint64)
        rc = lib().lc_sls_serialize_split_apsara_dev(
            self._h, ap._h, _p(d_src), src_len, _p(d_off), _p(d_len), n, _p(d_status), _p(d_sec), _p(d_nsec),
            _p(d_micro), _p(d_first), _p(d_entries),
            *self._sa_cfg(renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns,
                          enable_ns), _p(d_out), out_cap, C.byref(need), _p(ctr))
        if rc == LC_ERR_CAPACITY and d_out is None:
            return int(need.value), ctr  # a sizing query
        _check(rc)
        return int(need.value), ctr

    def _split_apsara(self, fn, ap, buf, extra, renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos,
                      time, time_ns, enable_ns, now, discard_interval, out_cap, ml, tail):
        """one host-buffer split -> Apsara call, sized by an estimate first and by the exact size when that was short;
        tail None: the wire bytes, else records ‖ tail as one LZ4 block.  Returns (bytes, raw_len, n_events,
        counters[5], ml_counters[3] or None)"""
        a = _u8(buf)
        cfg = self._sa_cfg(renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns,
                           enable_ns) + [int(now), int(discard_interval)]
        tl = None if tail is None else np.frombuffer(bytes(tail), np.uint8)
        est = 2 * a.size + 4096 + (0 if tl is None else tl.size)
        cap = int(out_cap if out_cap is not None else est + est // 255 + 16)
        for _ in range(2):
            out = np.empty(max(cap, 1), np.uint8)
            need, raw, nev = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
            ctr, mctr = np.zeros(5, np.uint64), np.zeros(3, np.uint64)
            z = [] if tl is None else [_p(tl) if tl.size else None, tl.size]
            outs = [_p(out), cap, C.byref(need)] + ([] if tl is None else [C.byref(raw)]) + [C.byref(nev), _p(ctr)]
            rc = fn(self._h, ap._h, _p(a), a.size, *extra, *cfg, *z, *outs, *([_p(mctr)] if ml else []))
            if rc == LC_ERR_CAPACITY and out_cap is None:
                cap = int(need.value)
                continue
            _check(rc)
            return bytes(out[:need.value]), int(raw.value), int(nev.value), ctr, (mctr if ml else None)
        _check(rc)

    def split_apsara_parse_sls(self, ap, buf, split_char, renamed_key, keep_fail=False, keep_succeed=False,
                               copy_raw=False, offset_key=None, src_pos=0, time=0, time_ns=None, enable_ns=False,
                               now=0, discard_interval=-1, out_cap=None):
        """Host source value in: split, Apsara (now, discard_interval -1 = no history discard), wire bytes out
        (lc_split_apsara_parse_sls).  Returns (bytes, number of pieces, counters[5])."""
        data, _raw, nev, ctr, _m = self._split_apsara(
            lib().lc_split_apsara_parse_sls, ap, buf, [split_char], renamed_key, keep_fail, keep_succeed, copy_raw,
            offset_key, src_pos, time, time_ns, enable_ns, now, discard_interval, out_cap, False, None)
        return data, nev, ctr

    def split_apsara_parse_sls_lz4(self, ap, buf, split_char, renamed_key, keep_fail=False, keep_succeed=False,
                                   copy_raw=False, offset_key=None, src_pos=0, time=0, time_ns=None, enable_ns=False,
                                   now=0, discard_interval=-1, tail=b"", out_cap=None):
        """split_apsara_parse_sls's records followed by `tail` as ONE LZ4 block (lc_split_apsara_parse_sls_lz4).
        Returns (block, raw_len, number of pieces, counters[5])."""
        data, raw, nev, ctr, _m = self._split_apsara(
            lib().lc_split_apsara_parse_sls_lz4, ap, buf, [split_char], renamed_key, keep_fail, keep_succeed,
            copy_raw, offset_key, src_pos, time, time_ns, enable_ns, now, discard_interval, out_cap, False, tail)
        return data, raw, nev, ctr

    def multiline_split_apsara_parse_sls(self, ap, buf, start, cont, end, discard, renamed_key, keep_fail=False,
                                         keep_succeed=False, copy_raw=False, offset_key=None, src_pos=0, time=0,
                                         time_ns=None, enable_ns=False, now=0, discard_interval=-1, out_cap=None):
        """The same with the multiline splitter (lc_multiline_split_apsara_parse_sls).  Returns (bytes, number of
        events, counters[5], splitter counters[3])."""
        data, _raw, nev, ctr, mctr = self._split_apsara(
            lib().lc_multiline_split_apsara_parse_sls, ap, buf, [_rh(start), _rh(cont), _rh(end), int(bool(discard))],
            renamed_key, keep_fail, keep_succeed, copy_raw, offset_key, src_pos, time, time_ns, enable_ns, now,
            discard_interval, out_cap, True, None)
        return data, nev, ctr, mctr

    def multiline_split_apsara_parse_sls_lz4(self, ap, buf, start, cont, end, discard, renamed_key, keep_fail=False,
                                             keep_succeed=False, copy_raw=False, offset_key=None, src_pos=0, time=0,
                                             time_ns=None, enable_ns=False, now=0, discard_interval=-1, tail=b"",
                                             out_cap=None):
        """multiline_split_apsara_parse_sls's records followed by `tail` as ONE LZ4 block
        (lc_multiline_split_apsara_parse_sls_lz4).  Returns (block, raw_len, number of events, counters[5], splitter
        counters[3])."""
        return self._split_apsara(
            lib().lc_multiline_split_apsara_parse_sls_lz4, ap, buf,
            [_rh(start), _rh(cont), _rh(end), int(bool(discard))], renamed_key, keep_fail, keep_succeed, copy_raw,
            offset_key, src_pos, time, time_ns, enable_ns, now, discard_interval, out_cap, True, tail)

    def json_parse_dev(self, js, d_base, base_len, d_ev_off, d_ev_len, n, d_status, d_first, d_entries, entry_cap,
                       d_arena, arena_cap, d_counters):
        """lc_json_parse_dev over device tables; waits for the device.  Returns (entry count, arena bytes); raises
        LcError with LC_ERR_CAPACITY when either exceeds its cap (nothing is written to the entries or the arena)."""
        m, ab = C.c_uint64(0), C.c_uint64(0)
        _check(lib().lc_json_parse_dev(self._h, js._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len), n,
                                       _p(d_status), _p(d_first), _p(d_entries), entry_cap, C.byref(m), _p(d_arena),
                                       arena_cap, C.byref(ab), _p(d_counters)))
        return m.value, ab.value

    def timestamp_parse_dev(self, ts, d_base, base_len, d_ev_off, d_ev_len, n, d_grp, ngroups, now, discard_interval,
                            d_sec, d_nsec, d_status, d_counters):
        _check(lib().lc_timestamp_parse_dev(self._h, ts._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len), n,
                                            _p(d_grp), ngroups, int(now), int(discard_interval), _p(d_sec), _p(d_nsec),
                                            _p(d_status), _p(d_counters)))

    def timestamp_parse_capture_dev(self, ts, d_base, base_len, d_rx_status, d_cap_off, d_cap_len, row_pitch, k, n,
                                    d_grp, ngroups, now, discard_interval, d_sec, d_nsec, d_status, d_counters):
        _check(lib().lc_timestamp_parse_capture_dev(self._h, ts._h, _p(d_base), base_len, _p(d_rx_status),
                                                    _p(d_cap_off), _p(d_cap_len), row_pitch, k, n, _p(d_grp), ngroups,
                                                    int(now), int(discard_interval), _p(d_sec), _p(d_nsec),
                                                    _p(d_status), _p(d_counters)))

    def regex_parse_dev(self, rx, d_base, base_len, d_ev_off, d_ev_len, n, nkeys, d_status, d_cap_off, d_cap_len):
        _check(lib().lc_regex_parse_dev(self._h, rx._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len), n, nkeys,
                                        _p(d_status), _p(d_cap_off), _p(d_cap_len)))

    def multiline_split_dev(self, d_buf, length, start, cont, end, discard, d_off, d_len, d_flags, cap):
        n = C.c_uint64(0)
        ctr = np.zeros(3, np.uint64)
        _check(lib().lc_multiline_split_dev(self._h, _p(d_buf), length, _rh(start), _rh(cont), _rh(end),
                                            int(bool(discard)), _p(d_off), _p(d_len), _p(d_flags), cap, C.byref(n),
                                            _p(ctr)))
        return n.value, ctr

    def delim_regex_chain(self, base, ev_off, ev_len, sep: bytes, quote, nkeys, extend, allow_short, max_fields, column,
                          rx, regex_nkeys=None):
        """Delimiter stage + regex stage on one column with host buffers (lc_delim_regex_chain); returns
        (status, nfields, f_off, f_len, f_dq, re_status, cap_off, cap_len)."""
        a = _u8(base)
        ev_off = np.ascontiguousarray(ev_off, np.uint32)
        ev_len = np.ascontiguousarray(ev_len, np.uint32)
        n, MF, G = ev_off.size, int(max_fields), rx.ngroups
        st, nf = np.empty(n, np.uint8), np.empty(n, np.uint32)
        fo, fl, fd = (np.empty((n, MF), np.uint32) for _ in range(3))
        rs = np.empty(n, np.uint8)
        co, cl = np.empty((n, G), np.uint32), np.empty((n, G), np.uint32)
        sp = np.frombuffer(sep, np.uint8)
        _check(lib().lc_delim_regex_chain(self._h, _p(a), a.size, _p(ev_off), _p(ev_len), n, _p(sp), len(sep), quote,
                                          nkeys, int(bool(extend)), int(bool(allow_short)), MF, _p(st), _p(nf), _p(fo),
                                          _p(fl), _p(fd), column, rx._h, G if regex_nkeys is None else regex_nkeys,
                                          _p(rs), _p(co), _p(cl)))
        return st, nf, fo, fl, fd, rs, co, cl

    def delim_parse_dev(self, d_base, base_len, d_ev_off, d_ev_len, n, sep: bytes, quote, nkeys, extend, allow_short,
                        max_fields, d_status, d_nf, d_fo, d_fl, d_fd, tap_col=None, d_tap_off=None, d_tap_len=None):
        sp = np.frombuffer(sep, np.uint8)
        _check(lib().lc_delim_parse_tap_dev(self._h, _p(d_base), base_len, _p(d_ev_off), _p(d_ev_len), n, _p(sp),
                                            len(sep), quote, nkeys, int(bool(extend)), int(bool(allow_short)),
                                            max_fields, _p(d_status), _p(d_nf), _p(d_fo), _p(d_fl), _p(d_fd),
                                            0xFFFFFFFF if tap_col is None else tap_col, _p(d_tap_off), _p(d_tap_len)))


class HostProcessor:
    """A GPU-backed Processor of the C++ host layer (include/lc_b200_host.h), driven with JSON event groups
    the way the reference's unit tests drive the original classes."""

    def __init__(self, ptype: str, config: dict):
        import json
        L = lib()
        L.lc_host_processor_create.restype = C.c_void_p
        L.lc_host_processor_create.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]
        L.lc_host_processor_destroy.argtypes = [C.c_void_p]
        L.lc_host_processor_process.restype = C.c_void_p
        L.lc_host_processor_process.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
        L.lc_host_processor_process_groups.restype = C.c_void_p
        L.lc_host_processor_process_groups.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]
        L.lc_host_processor_counters.restype = C.c_void_p
        L.lc_host_processor_counters.argtypes = [C.c_void_p]
        L.lc_host_string_free.argtypes = [C.c_void_p]
        err = C.c_void_p()
        self._h = L.lc_host_processor_create(ptype.encode(), json.dumps(config).encode("utf-8"), C.byref(err))
        if not self._h:
            msg = C.string_at(err.value).decode() if err.value else "unknown error"
            if err.value:
                L.lc_host_string_free(err)
            raise LcError(LC_ERR_INVALID_ARG, msg)
        self.type = ptype

    def process(self, group, enable_event_meta=True):
        """group: dict in the reference's event-group JSON shape (or None). Returns the processed group."""
        import json
        L = lib()
        err = C.c_void_p()
        out = L.lc_host_processor_process(self._h, json.dumps(group).encode("utf-8"), int(enable_event_meta),
                                          C.byref(err))
        if not out:
            msg = C.string_at(err.value).decode() if err.value else "unknown error"
            if err.value:
                L.lc_host_string_free(err)
            raise LcError(LC_ERR_CUDA, msg)
        s = C.string_at(out).decode("utf-8")
        L.lc_host_string_free(out)
        return json.loads(s)

    def process_groups(self, groups, enable_event_meta=True):
        """Processor::Process(std::vector<PipelineEventGroup>&) on a list of groups in one call.  Returns the list."""
        import json
        L = lib()
        err = C.c_void_p()
        out = L.lc_host_processor_process_groups(self._h, json.dumps(groups).encode("utf-8"), int(enable_event_meta),
                                                 C.byref(err))
        if not out:
            msg = C.string_at(err.value).decode() if err.value else "unknown error"
            if err.value:
                L.lc_host_string_free(err)
            raise LcError(LC_ERR_CUDA, msg)
        s = C.string_at(out).decode("utf-8")
        L.lc_host_string_free(out)
        return json.loads(s)

    def set_discard_old_data(self, enabled, interval=43200):
        """ilogtail_discard_old_data / ilogtail_discard_interval of a time-parsing processor"""
        L = lib()
        L.lc_host_processor_set_discard_old_data.argtypes = [C.c_void_p, C.c_int, C.c_int32]
        if L.lc_host_processor_set_discard_old_data(self._h, int(bool(enabled)), int(interval)) != 0:
            raise ValueError("not a time-parsing processor")

    def counters(self):
        import json
        L = lib()
        out = L.lc_host_processor_counters(self._h)
        s = C.string_at(out).decode()
        L.lc_host_string_free(out)
        return json.loads(s)

    def __del__(self):
        try:
            if self._h:
                lib().lc_host_processor_destroy(self._h)
        except Exception:
            pass


    def serialize_sls(self, group, enable_ns=False, process_then_serialize=False):
        """SerializeSls of a processor_parse_delimiter_native, processor_parse_regex_native, processor_split_string_native
        or processor_split_multiline_log_string_native on a JSON group: (bytes, None) or (None, error).  With process_then_serialize, Process + SLSEventGroupSerializer::Serialize on the same
        in-memory group instead."""
        import json
        L = lib()
        L.lc_host_processor_serialize_sls.restype = C.c_void_p
        L.lc_host_processor_serialize_sls.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int,
                                                      C.POINTER(C.c_ulonglong), C.POINTER(C.c_void_p),
                                                      C.POINTER(C.c_void_p)]
        L.lc_host_string_free.argtypes = [C.c_void_p]
        err = C.c_void_p()
        fail = C.c_void_p()
        n = C.c_ulonglong(0)
        out = L.lc_host_processor_serialize_sls(self._h, json.dumps(group).encode("utf-8"), int(bool(enable_ns)),
                                                int(bool(process_then_serialize)), C.byref(n), C.byref(err),
                                                C.byref(fail))
        if fail.value:
            msg = C.string_at(fail.value).decode()
            L.lc_host_string_free(fail)
            raise LcError(LC_ERR_CUDA, msg)
        if not out:
            msg = C.string_at(err.value).decode() if err.value else "unknown error"
            if err.value:
                L.lc_host_string_free(err)
            return None, msg
        data = C.string_at(out, n.value)
        L.lc_host_string_free(out)
        return data, None

    def serialize_sls_lz4(self, group, enable_ns=False):
        """SerializeSlsLz4 of a processor_parse_delimiter_native or processor_parse_regex_native on a JSON group:
        (block, raw_len, None) or (None, 0, error)."""
        import json
        L = lib()
        L.lc_host_processor_serialize_sls_lz4.restype = C.c_void_p
        L.lc_host_processor_serialize_sls_lz4.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.POINTER(C.c_ulonglong),
                                                          C.POINTER(C.c_ulonglong), C.POINTER(C.c_void_p),
                                                          C.POINTER(C.c_void_p)]
        L.lc_host_string_free.argtypes = [C.c_void_p]
        err, fail = C.c_void_p(), C.c_void_p()
        n, raw = C.c_ulonglong(0), C.c_ulonglong(0)
        out = L.lc_host_processor_serialize_sls_lz4(self._h, json.dumps(group).encode("utf-8"), int(bool(enable_ns)),
                                                    C.byref(n), C.byref(raw), C.byref(err), C.byref(fail))
        if fail.value:
            msg = C.string_at(fail.value).decode()
            L.lc_host_string_free(fail)
            raise LcError(LC_ERR_CUDA, msg)
        if not out:
            msg = C.string_at(err.value).decode() if err.value else "unknown error"
            if err.value:
                L.lc_host_string_free(err)
            return None, 0, msg
        data = C.string_at(out, n.value)
        L.lc_host_string_free(out)
        return data, int(raw.value), None


def host_chain_serialize_sls(delim, regex, group, enable_ns=False, mode=0):
    """The delimiter -> regex, split -> regex or split -> delimiter chain of two HostProcessors on a JSON group
    (lc_host_chain_serialize_sls; delim may be either splitter, and regex a delimiter behind a splitter).  mode 0:
    delim's SerializeSls(group, regex); 1: Process + Process + Serialize; 2: SerializeSlsLz4.  Returns (bytes, raw_len,
    None) or (None, 0, error)."""
    import json
    L = lib()
    L.lc_host_chain_serialize_sls.restype = C.c_void_p
    L.lc_host_chain_serialize_sls.argtypes = [C.c_void_p, C.c_void_p, C.c_char_p, C.c_int, C.c_int,
                                              C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong),
                                              C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    L.lc_host_string_free.argtypes = [C.c_void_p]
    err, fail = C.c_void_p(), C.c_void_p()
    n, raw = C.c_ulonglong(0), C.c_ulonglong(0)
    out = L.lc_host_chain_serialize_sls(delim._h, regex._h, json.dumps(group).encode("utf-8"), int(bool(enable_ns)),
                                        mode, C.byref(n), C.byref(raw), C.byref(err), C.byref(fail))
    if fail.value:
        msg = C.string_at(fail.value).decode()
        L.lc_host_string_free(fail)
        raise LcError(LC_ERR_CUDA, msg)
    if not out:
        msg = C.string_at(err.value).decode() if err.value else "unknown error"
        if err.value:
            L.lc_host_string_free(err)
        return None, 0, msg
    data = C.string_at(out, n.value)
    L.lc_host_string_free(out)
    return data, int(raw.value), None


def host_chain3_serialize_sls(split, regex, filt, group, enable_ns=False, mode=0):
    """The split -> regex -> filter chain of three HostProcessors on a JSON group (lc_host_chain3_serialize_sls).
    mode 0: split's SerializeSls(group, regex, filter); 1: Process x 3 + Serialize; 2: SerializeSlsLz4.  Returns (bytes,
    raw_len, None) or (None, 0, error).  The split -> delimiter -> regex chain goes through the same call, with a
    delimiter processor as `regex` and a regex processor as `filt`; so does the split -> regex -> timestamp chain, with
    a timestamp processor as `filt`."""
    import json
    L = lib()
    L.lc_host_chain3_serialize_sls.restype = C.c_void_p
    L.lc_host_chain3_serialize_sls.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int, C.c_int,
                                               C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong),
                                               C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    L.lc_host_string_free.argtypes = [C.c_void_p]
    err, fail = C.c_void_p(), C.c_void_p()
    n, raw = C.c_ulonglong(0), C.c_ulonglong(0)
    out = L.lc_host_chain3_serialize_sls(split._h, regex._h, filt._h, json.dumps(group).encode("utf-8"),
                                         int(bool(enable_ns)), mode, C.byref(n), C.byref(raw), C.byref(err),
                                         C.byref(fail))
    if fail.value:
        msg = C.string_at(fail.value).decode()
        L.lc_host_string_free(fail)
        raise LcError(LC_ERR_CUDA, msg)
    if not out:
        msg = C.string_at(err.value).decode() if err.value else "unknown error"
        if err.value:
            L.lc_host_string_free(err)
        return None, 0, msg
    data = C.string_at(out, n.value)
    L.lc_host_string_free(out)
    return data, int(raw.value), None


def host_lz4_compress(inputs):
    """The host layer's GPU-backed LZ4Compressor::Compress over a list of byte strings in one device call
    (lc_host_lz4_compress): (list of blocks, None) or (None, error)."""
    L = lib()
    L.lc_host_lz4_compress.restype = C.c_void_p
    L.lc_host_lz4_compress.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.POINTER(C.c_ulonglong), C.c_void_p,
                                       C.POINTER(C.c_void_p)]
    L.lc_host_string_free.argtypes = [C.c_void_p]
    bufs = [bytes(x) for x in inputs]
    n = len(bufs)
    ptrs = (C.c_char_p * max(n, 1))(*bufs)
    lens = np.array([len(b) for b in bufs] or [0], np.uint64)
    blen = np.zeros(max(n, 1), np.uint64)
    total, err = C.c_ulonglong(0), C.c_void_p()
    out = L.lc_host_lz4_compress(C.cast(ptrs, C.c_void_p), _p(lens), n, C.byref(total), _p(blen), C.byref(err))
    if not out:
        msg = C.string_at(err.value).decode() if err.value else "unknown error"
        if err.value:
            L.lc_host_string_free(err)
        return None, msg
    data = C.string_at(out, total.value)
    L.lc_host_string_free(out)
    res, o = [], 0
    for k in range(n):
        res.append(data[o:o + int(blen[k])])
        o += int(blen[k])
    return res, None


def zstd_bound(n):
    """ZSTD_compressBound(n): the largest frame lc_zstd_compress[_dev] makes of n bytes."""
    return n + (n >> 8) + (((128 << 10) - n) >> 11 if n < (128 << 10) else 0)


def host_zstd_compress(inputs):
    """The host layer's GPU-backed ZstdCompressor::Compress over a list of byte strings in one device call
    (lc_host_zstd_compress): (list of frames, None) or (None, error)."""
    L = lib()
    L.lc_host_zstd_compress.restype = C.c_void_p
    L.lc_host_zstd_compress.argtypes = [C.c_void_p, C.c_void_p, C.c_ulonglong, C.POINTER(C.c_ulonglong), C.c_void_p,
                                        C.POINTER(C.c_void_p)]
    L.lc_host_string_free.argtypes = [C.c_void_p]
    bufs = [bytes(x) for x in inputs]
    n = len(bufs)
    ptrs = (C.c_char_p * max(n, 1))(*bufs)
    lens = np.array([len(b) for b in bufs] or [0], np.uint64)
    flen = np.zeros(max(n, 1), np.uint64)
    total, err = C.c_ulonglong(0), C.c_void_p()
    out = L.lc_host_zstd_compress(C.cast(ptrs, C.c_void_p), _p(lens), n, C.byref(total), _p(flen), C.byref(err))
    if not out:
        msg = C.string_at(err.value).decode() if err.value else "unknown error"
        if err.value:
            L.lc_host_string_free(err)
        return None, msg
    data = C.string_at(out, total.value)
    L.lc_host_string_free(out)
    res, o = [], 0
    for k in range(n):
        res.append(data[o:o + int(flen[k])])
        o += int(flen[k])
    return res, None


def host_sls_serialize(group, enable_ns=False):
    """SLSEventGroupSerializer::Serialize of the C++ host layer on a JSON event group: (bytes, None) or (None, error)."""
    import json
    L = lib()
    L.lc_host_sls_serialize.restype = C.c_void_p
    L.lc_host_sls_serialize.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_ulonglong), C.POINTER(C.c_void_p)]
    L.lc_host_string_free.argtypes = [C.c_void_p]
    err = C.c_void_p()
    n = C.c_ulonglong(0)
    out = L.lc_host_sls_serialize(json.dumps(group).encode("utf-8"), int(bool(enable_ns)), C.byref(n), C.byref(err))
    if not out:
        msg = C.string_at(err.value).decode() if err.value else "unknown error"
        if err.value:
            L.lc_host_string_free(err)
        return None, msg
    data = C.string_at(out, n.value)
    L.lc_host_string_free(out)
    return data, None
