"""In-tree build of libloongcollector_b200.so (nvcc, sm_90a only: H100).

The shared object lands next to this file, so that the package is importable from the source tree
(it is git-ignored)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libloongcollector_b200.so")
SOURCES = ["regex_compiler.cpp", "lc_kernels.cu", "lc_capi.cu"]
HEADERS = ["lc_tables.h", "lc_json_pow5.h", "lc_exec.cuh", "lc_scan.cuh", "lc_kernels.cuh", "regex_compiler.h",
           os.path.join("..", "..", "include", "lc_b200.h")]
HOST_DIR = os.path.join(HERE, "host")

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xptxas", "-v",
]


def _host_sources():
    if not os.path.isdir(HOST_DIR):
        return []
    return sorted(os.path.join(HOST_DIR, f) for f in os.listdir(HOST_DIR) if f.endswith((".cpp", ".cu")))


def _host_headers():
    if not os.path.isdir(HOST_DIR):
        return []
    return sorted(os.path.join(HOST_DIR, f) for f in os.listdir(HOST_DIR) if f.endswith((".h", ".cuh")))


def needs_build():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + _host_sources() + _host_headers() + [__file__] + \
        [os.path.join(PLUGIN_DIR, "dynamic_processor.cpp")]
    if not all(os.path.exists(plugin_path(n)) for n, _ in PLUGINS):
        return True
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


# dynamic plugins (plugin/dynamic_processor.cpp): one .so per processor, named lib<name>.so as the agent's loader expects
PLUGIN_DIR = os.path.join(HERE, "plugin")
PLUGINS = [
    ("processor_parse_regex_b200", "processor_parse_regex_native"),
    ("processor_parse_delimiter_b200", "processor_parse_delimiter_native"),
    ("processor_split_string_b200", "processor_split_string_native"),
    ("processor_split_multiline_log_string_b200", "processor_split_multiline_log_string_native"),
]


def plugin_path(name):
    return os.path.join(PLUGIN_DIR, "lib%s.so" % name)


def build_plugins(log):
    gxx = os.environ.get("CXX", "g++")
    src = os.path.join(PLUGIN_DIR, "dynamic_processor.cpp")
    for name, ptype in PLUGINS:
        cmd = [gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-DLC_PLUGIN_NAME=\"%s\"" % name,
               "-DLC_PLUGIN_TYPE=\"%s\"" % ptype, src, "-o", plugin_path(name), "-L", HERE,
               "-l:libloongcollector_b200.so", "-Wl,-rpath,$ORIGIN/.."]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        log.write(" ".join(cmd) + "\n" + p.stdout)
        if p.returncode != 0:
            sys.stderr.write(p.stdout)
            raise RuntimeError("plugin build failed: %s" % name)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-I", CSRC, "-I", os.path.join(HERE, "..", "include")] + \
        [os.path.join(CSRC, s) for s in SOURCES] + _host_sources() + ["-o", SO]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log = os.path.join(HERE, "build.log")
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + p.stdout)
        if p.returncode == 0:
            build_plugins(f)
    if verbose or p.returncode != 0:
        sys.stderr.write(p.stdout)
    if p.returncode != 0:
        raise RuntimeError("nvcc failed (see %s)" % log)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
