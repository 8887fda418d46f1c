"""CPU tier: the kernels' run-skipping delimiter state machine (csrc/lc_exec.cuh: lc_delim_fsm, compiled for the
host by tests/emul) against the oracle's per-byte restatement of DelimiterModeFsmParser::ParseDelimiterLine -- every
column (offset, length, doubled-quote count), the column count and the error verdict, on well-formed and malformed
lines, at every 16-byte alignment and for sub-ranges (the processor trims blanks first)."""
import ctypes as C
import random

import numpy as np

from oracle import oracle as orc
from tests.emul import emul


def _oracle(line: bytes, begin: int, end: int, sep: int, quote: int, cap: int):
    a = np.frombuffer(line, np.uint8) if line else np.zeros(1, np.uint8)
    fo = np.zeros(cap, np.uint32)
    fl = np.zeros(cap, np.uint32)
    fd = np.zeros(cap, np.uint32)
    n = orc.lib().orc_delim_fsm(a.ctypes.data_as(C.c_void_p), begin, end, sep, quote, fo.ctypes.data_as(C.c_void_p),
                                fl.ctypes.data_as(C.c_void_p), fd.ctypes.data_as(C.c_void_p), cap)
    if n < 0:
        return None
    k = min(int(n), cap)
    return int(n), list(zip(fo[:k].tolist(), fl[:k].tolist(), fd[:k].tolist()))


def _rand_line(rng, alphabet, lo, hi):
    return bytes(rng.choices(alphabet, k=rng.randint(lo, hi)))


# the blank as separator and as quote (both interact with the processor's trim), next to the usual pairs
CONFIGS = ((ord(","), ord('"')), (ord("|"), ord("'")), (ord("\t"), ord('"')), (ord(" "), ord('"')),
           (ord(","), ord(" ")))


def _long_fields(sep, quote):
    """fields of 31, 33 and 200 bytes, plain and quoted (with separators and doubled quotes inside): one 32-byte step of
    the kernels and either side of it, and a field over more than one 128-byte stage"""
    q, s = bytes([quote]), bytes([sep])
    out = []
    for n in (31, 33, 200):
        body = (b"0123456789abcdefxyz" * 11)[:n]
        out += [body, q + body[:n - 2] + q, q + (s + q * 2 + body)[:n - 2] + q]
    return out


def test_run_skipping_fsm_equals_per_byte_fsm():
    rng = random.Random(4242)
    checked = errors = 0
    for sep, quote in CONFIGS:
        soup = bytes([sep, sep, quote, quote]) + b"abc d0123456789xyz"
        wellformed_fields = [b"", b"a", b"abc", b"0123456789abcdefghij",
                             bytes([quote]) + b"q" + bytes([sep]) + b"x" + bytes([quote]),
                             bytes([quote, quote, quote]) + b"in" + bytes([quote, quote, quote]),
                             bytes([quote, quote])] + _long_fields(sep, quote)
        for it in range(6000):
            if it % 3 == 0:
                line = bytes([sep]).join(rng.choice(wellformed_fields) for _ in range(rng.randint(1, 14)))[:400]
            else:
                line = _rand_line(rng, soup, 0, 400 if it % 3 == 1 else 70)
            if not line:
                continue
            pad = rng.randint(16, 31)  # every alignment of the line start within a 16-byte chunk
            buf = np.zeros(pad + len(line) + 48, np.uint8)
            buf[:pad] = rng.choice([sep, quote, 65])  # neighbours must not leak into the result
            buf[pad + len(line):] = rng.choice([sep, quote, 66])
            buf[pad:pad + len(line)] = np.frombuffer(line, np.uint8)
            begin = rng.randint(0, min(3, len(line) - 1)) if rng.random() < 0.3 else 0
            end = rng.randint(begin + 1, len(line)) if rng.random() < 0.3 else len(line)
            cap = rng.choice([2, 5, 64])
            want = _oracle(line, begin, end, sep, quote, cap)
            got = emul.delim_fsm(buf, pad, begin, end, sep, quote, cap)
            assert got == want, (line, begin, end, sep, quote, cap, got, want)
            checked += 1
            errors += want is None
    assert checked > 15000 and errors > 1000


def test_bit_parallel_path_equals_the_machine_where_it_applies():
    """lc_delim_fast either produces the machine's columns or hands the record over; it must take the records in which
    every quote is one the machine accepts, and never claim an erroneous one."""
    rng = random.Random(99)
    taken = handed = 0
    for sep, quote in CONFIGS:
        soup = bytes([sep, sep, quote, quote]) + b"abc d0123456789xyz"
        q = bytes([quote])
        wellformed_fields = [b"", b"a", b"abc", b"0123456789abcdefghij", b"a b  c", q + b"q" + bytes([sep]) + b"x" + q,
                             q * 3 + b"in" + q * 3, q * 2, q * 4, q + b"0123456789abcdef" + q, q + b"a" + q * 2 + b"b" + q,
                             q + bytes([sep]) * 3 + q]
        wellformed_fields += _long_fields(sep, quote)
        for it in range(8000):
            if it % 2 == 0:
                line = bytes([sep]).join(rng.choice(wellformed_fields) for _ in range(rng.randint(1, 14)))[:400]
            else:
                line = _rand_line(rng, soup, 0, 400 if it % 4 == 1 else 70)
            if not line:
                continue
            pad = rng.randint(16, 31)
            buf = np.zeros(pad + len(line) + 48, np.uint8)
            buf[:pad] = rng.choice([sep, quote, 65])
            buf[pad + len(line):] = rng.choice([sep, quote, 66])
            buf[pad:pad + len(line)] = np.frombuffer(line, np.uint8)
            begin = rng.randint(0, min(3, len(line) - 1)) if rng.random() < 0.3 else 0
            end = rng.randint(begin + 1, len(line)) if rng.random() < 0.3 else len(line)
            cap = rng.choice([2, 5, 64])
            want = _oracle(line, begin, end, sep, quote, cap)
            got = emul.delim_fast(buf, pad, begin, end, sep, quote, cap)
            if got is None:
                handed += 1
                # whatever the machine accepts is well-formed in the sense of the fast path: it must not hand it over
                assert want is None, (line, begin, end, sep, quote, want)
                continue
            taken += 1
            assert want is not None, (line, begin, end, sep, quote, got)
            n, fo, fl, fd = got
            assert (n, list(zip(fo.tolist(), fl.tolist(), fd.tolist()))) == want, (line, begin, end, sep, quote, cap,
                                                                                    got, want)
    assert taken > 11000 and handed > 1500
