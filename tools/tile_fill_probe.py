"""Tile fill probe: times the line loader's stage loop alone (tile_fill_probe.cu) with the chunk-major and the
line-major layout of the staging tile, over C2's line shape (4 Mi lines x 256 B), with line starts 128-byte aligned
and 16 bytes in, once with the lines resident in HBM and once with a 16 MB working set that stays in L2 (there the
fill is not bound by HBM, so a difference on the shared-memory side shows).

  python tools/tile_fill_probe.py [--reps N]

Prints one JSON line: card name, power limit, SM clock limit, and per layout and placement the median / min / max
kernel time in ms (CUDA events, the two layouts alternating launch by launch)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))

from loongcollector_b200 import _build  # noqa: E402

LINES, PITCH = 4 << 20, 256
L2_LINES = 64 << 10  # 16 MB: well inside the H100's 50 MB L2


def nvidia_smi(query):
    try:
        p = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + query, "--format=csv,noheader,nounits"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return [x.strip() for x in p.stdout.strip().split(",")]
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    flags = [f for f in _build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "tile_fill_probe")
        subprocess.run([nvcc] + flags + [os.path.join(HERE, "tile_fill_probe.cu"), "-o", exe], check=True,
                       stdout=subprocess.DEVNULL)
        res = {}
        for ws_name, ws in (("hbm", LINES), ("l2", L2_LINES)):
            out = subprocess.run([exe, str(LINES), str(PITCH), str(args.reps), str(ws)], check=True,
                                 stdout=subprocess.PIPE, text=True).stdout
            for ln in out.strip().splitlines():
                f = ln.split()
                t = [float(x) for x in f[4:]]
                res["%s/%s/%s" % (ws_name, f[1], f[0])] = {
                    "median_ms": round(statistics.median(t), 5), "min_ms": min(t), "max_ms": max(t), "n": len(t)}
    card = nvidia_smi("name,power.limit,clocks.max.sm")
    line = {"probe": "tile_fill", "lines": LINES, "pitch": PITCH, "card": card[0] if card else None,
            "power_limit_w": card[1] if card else None, "sm_max_mhz": card[2] if card else None, "results": res}
    for k in list(res):
        if k.endswith("/chunk_major"):
            lm = res[k[:-len("chunk_major")] + "line_major"]
            res[k[:-len("/chunk_major")] + "/speedup"] = round(res[k]["median_ms"] / lm["median_ms"], 4)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
