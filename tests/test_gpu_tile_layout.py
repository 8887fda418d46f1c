"""GPU tier: the staging tile of the line loader (lc_kernels.cu: tile_slot, TdfaLoader) in every kernel that uses it --
regex_tdfa_staged_kernel, regex_tdfa_multi_kernel and delim_tiled_kernel -- against the CPU oracle.

Line lengths put 0..8 chunks into a line's last stage, mixed inside one warp; line starts fall on every 16-byte offset
of a 128-byte line and the arena base is misaligned by 0..15 bytes; batch sizes are not multiples of 32; lines die in
the first stage next to lines that run to the end; a multi-pattern batch has lanes that matched an earlier pattern;
delimiter records put a separator or a quote into every byte of the two chunks the kernel reads per step."""
import random

import numpy as np
import pytest

from oracle import oracle as orc  # checker only

pytestmark = pytest.mark.gpu

SIMPLE = r'(\w+) "([^"]*)" (\d+)(.*)'


@pytest.fixture(scope="module")
def lc():
    import loongcollector_b200
    return loongcollector_b200


@pytest.fixture(scope="module")
def eng(lc):
    e = lc.Engine(0)
    yield e
    e.close()


def _simple_line(rng, n):
    """A line of exactly n bytes: matches SIMPLE when long enough, most of its bytes inside [^"]* (run skipping)."""
    if n < 8 or rng.random() < 0.15:
        return bytes(rng.choice(b' #"ab1') for _ in range(n))  # mostly dies at once
    quoted = max(0, n - 8 - rng.randint(0, min(24, n - 8)))
    s = b"k " + b'"' + bytes(rng.choice(b"abc /-x") for _ in range(quoted)) + b'" 7'
    return (s + b"t" * n)[:n]


def _lengths(rng, count):
    """Lengths whose last stage (128 bytes) holds 0..8 chunks for every start offset, shuffled so a warp mixes them."""
    out = [rng.choice((0, 1, 2, 15, 16, 17)) for _ in range(count // 8)]
    while len(out) < count:
        stages = rng.randint(0, 2)
        out.append(stages * 128 + rng.randint(0, 128))
    rng.shuffle(out)
    return out


def _arena(lines, lead, pad_to=16):
    """lines laid out behind `lead` filler bytes (sets the 128-byte phase of every start), plus a guard tail."""
    base = b"\x00" * lead + b"".join(lines) + b"\x00" * pad_to
    ln = np.array([len(x) for x in lines], np.uint32)
    off = np.zeros(len(lines), np.uint32)
    off[:] = lead + np.concatenate(([0], np.cumsum(ln[:-1]))) if len(lines) else 0
    return np.frombuffer(base, np.uint8), off, ln


def _regex_dev(lc, eng, rx, nkeys, buf, off, ln, shift):
    """lc_regex_parse_dev with the arena starting `shift` bytes past a 256-byte aligned device address."""
    import torch
    dev = torch.device("cuda", 0)
    n, G = off.size, rx.ngroups
    t = torch.zeros(buf.size + 512, dtype=torch.uint8, device=dev)
    t[shift:shift + buf.size] = torch.from_numpy(buf.copy()).to(dev)
    d_off = torch.from_numpy(off.astype(np.int32)).to(dev)
    d_len = torch.from_numpy(ln.astype(np.int32)).to(dev)
    d_st = torch.zeros(n, dtype=torch.uint8, device=dev)
    d_co = torch.zeros(max(1, n * G), dtype=torch.int32, device=dev)
    d_cl = torch.zeros(max(1, n * G), dtype=torch.int32, device=dev)
    eng.regex_parse_dev(rx, t.data_ptr() + shift, buf.size, d_off.data_ptr(), d_len.data_ptr(), n, nkeys,
                        d_st.data_ptr(), d_co.data_ptr(), d_cl.data_ptr())
    torch.cuda.synchronize()
    co = d_co.cpu().numpy().view(np.uint32)[:n * G].reshape(n, G)
    cl = d_cl.cpu().numpy().view(np.uint32)[:n * G].reshape(n, G)
    return d_st.cpu().numpy(), co, cl


@pytest.mark.parametrize("shift", range(16))
def test_regex_staged_every_last_stage_fill_and_start_offset(lc, eng, shift):
    rng = random.Random(100 + shift)
    rx, orx = lc.Regex(SIMPLE), orc.Regex(SIMPLE)
    nkeys = rx.ngroups
    for lead in range(0, 128, 16):
        n = 32 * rng.randint(3, 6) + rng.randint(1, 31)
        lines = [_simple_line(rng, k) for k in _lengths(rng, n)]
        buf, off, ln = _arena(lines, lead)
        st, co, cl = _regex_dev(lc, eng, rx, nkeys, buf, off, ln, shift)
        est, eco, ecl = orc.regex_parse_batch(orx, buf, off, ln, nkeys)
        assert np.array_equal(st, est), (lead, np.nonzero(st != est)[0][:5])
        assert np.array_equal(co, eco[:, :rx.ngroups]) and np.array_equal(cl, ecl[:, :rx.ngroups]), lead
        assert (est == 0).any() and (est == 1).any()


def test_regex_staged_nginx_lines_at_every_offset(lc, eng):
    from loongcollector_b200 import synth
    rng = random.Random(7)
    rx, orx = lc.Regex(synth.NGINX_PATTERN), orc.Regex(synth.NGINX_PATTERN)
    lines = [synth._nginx_line(rng, target_len=rng.randint(110, 400), bad=rng.random() < 0.1).encode()
             for _ in range(32 * 9 + 5)]
    for lead in range(0, 144, 9):
        buf, off, ln = _arena(lines, lead)
        st, co, cl = eng.regex_parse(rx, buf, off, ln, 10)
        est, eco, ecl = orc.regex_parse_batch(orx, buf, off, ln, 10)
        assert np.array_equal(st, est), (lead, np.nonzero(st != est)[0][:5])
        assert np.array_equal(co, eco[:, :rx.ngroups]) and np.array_equal(cl, ecl[:, :rx.ngroups]), lead


def test_regex_multi_with_lanes_matched_by_an_earlier_pattern(lc, eng):
    from loongcollector_b200 import synth
    rng = random.Random(11)
    pats = [synth.NGINX_PATTERN, SIMPLE, r"(\S+) (\S+)(.*)"]
    nkeys = [10, 4, 3]
    lines = []
    for k in _lengths(rng, 32 * 12 + 19):
        r = rng.random()
        lines.append(synth._nginx_line(rng, target_len=max(110, k)).encode() if r < 0.3 else _simple_line(rng, k))
    rxs, orxs = [lc.Regex(p) for p in pats], [orc.Regex(p) for p in pats]
    for lead in (0, 5, 16, 48, 77, 112):
        buf, off, ln = _arena(lines, lead)
        which, status, co, cl = eng.regex_parse_multi(rxs, nkeys, buf, off, ln)
        gmax = max(r.ngroups for r in rxs)
        ewhich = np.full(off.size, 0xFF, np.uint8)
        est = np.ones(off.size, np.uint8)
        eco = np.zeros((off.size, gmax), np.uint32)
        ecl = np.zeros((off.size, gmax), np.uint32)
        for p, (o, k) in enumerate(zip(orxs, nkeys)):
            s, c, l = orc.regex_parse_batch(o, buf, off, ln, k)
            take = (ewhich == 0xFF) & (s != 1)
            ewhich[take], est[take] = p, s[take]
            ok = take & (s == 0)
            eco[ok, :o.ngroups] = c[ok, :o.ngroups]
            ecl[ok, :o.ngroups] = l[ok, :o.ngroups]
        assert len(set(ewhich.tolist())) >= 3  # lanes of one batch finish at different patterns
        assert np.array_equal(which, ewhich) and np.array_equal(status, est), lead
        assert np.array_equal(co, eco) and np.array_equal(cl, ecl), lead


@pytest.mark.parametrize("special", [b",", b'"'])
def test_delim_tiled_special_byte_in_every_slot_of_a_step(eng, special):
    """delim_tiled_kernel reads chunks k and k + 1 per 32-byte step: a separator or a quote at every byte of both, at
    every start offset of a 128-byte line."""
    rng = random.Random(3 if special == b"," else 4)
    lines = []
    for p in range(0, 160):
        for _ in range(2):
            n = rng.randint(p + 1, p + 40)
            s = bytearray(rng.choice(b"abcxyz019") for _ in range(n))
            if special == b'"':  # a quoted column that starts at p and closes a few bytes later (or stays open)
                s[p] = ord('"')
                q = p + rng.randint(1, 20)
                if q < n and rng.random() < 0.8:
                    s[q] = ord('"')
                    if q + 1 < n:
                        s[q + 1] = ord(",")
            else:
                s[p] = ord(",")
            lines.append(bytes(s))
    rng.shuffle(lines)
    lines = lines[:32 * 9 + 7]
    for lead in range(0, 128, 7):
        buf, off, ln = _arena(lines, lead)
        got = eng.delim_parse(buf, off, ln, b",", ord('"'), 6, True, True, 8)
        want = orc.delim_parse_batch(buf, off, ln, b",", ord('"'), 6, True, True, 8)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), (special, lead)
