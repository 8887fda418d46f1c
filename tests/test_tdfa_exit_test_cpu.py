"""CPU tier: lc_tdfa_chunk_has_exit (lc_exec.cuh), the branch-free run-skip test of the tagged-DFA walk, against the
per-exit loop it replaced, on skip words as regex_compiler.cpp encodes them (a one-exit state repeats its byte): 0, 1 and
2 exits, exit bytes 0x00, 0x80, 0xFF and others, the exit at each of the 16 positions of a chunk, and no exit at all."""
import os
import shutil
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "loongcollector_b200", "csrc")

PROGRAM = r"""
#include <cstdio>
#include <cstring>
#include "lc_exec.cuh"

static bool loop_has_exit(uint32_t sk, const uint32_t w[4]) { // the per-exit loop the kernels ran before
    const uint32_t n = (sk >> 16) & 3u;
    uint32_t hit = 0;
    for (uint32_t k = 0; k < n; ++k) {
        const uint32_t splat = ((sk >> (8 * k)) & 0xFFu) * 0x01010101u;
        for (int j = 0; j < 4; ++j) {
            const uint32_t x = w[j] ^ splat;
            hit |= (x - 0x01010101u) & ~x & 0x80808080u;
        }
    }
    return hit != 0;
}

int main() {
    const unsigned bytes[] = {0x00, 0x01, 0x22, 0x5C, 0x7F, 0x80, 0xFE, 0xFF};
    const unsigned fill[] = {0x00, 0x20, 0x61, 0xFF};
    long cases = 0, bad = 0, hits = 0;
    for (unsigned nexit = 0; nexit <= 2; ++nexit)
        for (unsigned a : bytes)
            for (unsigned b : bytes) {
                if (nexit < 2 && b != bytes[0]) continue;
                const unsigned e0 = nexit ? a : 0, e1 = nexit == 2 ? b : nexit == 1 ? a : 0;
                const uint32_t sk = LC_TDFA_SKIP | nexit << 16 | e1 << 8 | e0;
                for (unsigned f : fill)
                    for (int pos = -1; pos < 16; ++pos)          // -1: no planted byte
                        for (unsigned planted : bytes) {
                            uint8_t c[16];
                            memset(c, (int)f, 16);
                            if (pos >= 0) c[pos] = (uint8_t)planted;
                            uint32_t w[4];
                            memcpy(w, c, 16);
                            const bool want = loop_has_exit(sk, w), got = lc_tdfa_chunk_has_exit(sk, w);
                            ++cases;
                            hits += want;
                            if (want != got) {
                                if (++bad <= 5)
                                    printf("sk=%08x fill=%02x pos=%d byte=%02x want=%d got=%d\n", sk, f, pos, planted,
                                           want, got);
                            }
                        }
            }
    printf("cases=%ld hits=%ld bad=%ld\n", cases, hits, bad);
    return bad != 0 || hits == 0 || hits == cases;
}
"""


@pytest.mark.skipif(shutil.which(os.environ.get("CXX", "g++")) is None, reason="needs a C++ compiler")
def test_branch_free_exit_test_equals_the_loop(tmp_path):
    src = tmp_path / "exit_test.cpp"
    src.write_text(PROGRAM)
    exe = tmp_path / "exit_test"
    subprocess.run([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-I", CSRC, str(src), "-o", str(exe)],
                   check=True)
    p = subprocess.run([str(exe)], stdout=subprocess.PIPE, text=True)
    assert p.returncode == 0, p.stdout
