"""GPU tier: run skipping in the tagged-DFA walk (lc_kernels.cu: tdfa_walk_lines) is decided once per warp.  A chunk
is skipped only when every walking lane is in a skippable state and none of them finds an exit byte in it; otherwise
all walking lanes walk it.  These 32-line batches put the warp on each side of that vote, in both
regex_tdfa_staged_kernel and regex_tdfa_multi_kernel, against the CPU oracle:

* all lanes inside a [^"]* run, and all but one;
* one lane whose closing quote falls on each of the 16 byte slots of a chunk while the others stay in the run;
* dead lanes (lines that die at once or after a few bytes) mixed with live ones;
* ragged lengths with every start misalignment 0..15 inside one warp;
* with the length-order pre-pass off and forced on (which regroups the lines into other warps)."""
import random

import numpy as np
import pytest

from oracle import oracle as orc  # checker only

pytestmark = pytest.mark.gpu

SIMPLE = r'(\w+) "([^"]*)" (\d+)(.*)'
RUN = b"abc /-x.:="  # bytes that keep [^"]* in its state


@pytest.fixture(scope="module")
def lc():
    import loongcollector_b200
    return loongcollector_b200


def _quoted(rng, n, close_at=None):
    """A line of n bytes matching SIMPLE whose quoted field runs from byte 3 to `close_at` (default: near the end)."""
    if close_at is None:
        close_at = max(3, n - 4 - rng.randint(0, 3))
    s = b'k "' + bytes(rng.choice(RUN) for _ in range(close_at - 3)) + b'" 7'
    return (s + bytes(rng.choice(b"tu") for _ in range(n)))[:n]


def _word(rng, n):
    """A line of n bytes whose first 3/4 are one \\w+ run: a state that cannot skip."""
    w = max(1, 3 * n // 4)
    s = b"a" * w + b' "x" 1'
    return (s + b"z" * n)[:n]


def _dies(rng, n):
    """A line that kills the automaton at once or after a few bytes."""
    return (rng.choice((b"#", b"k x", b'kk "ab" q')) + b"y" * n)[:n]


def _batches(rng):
    """List of 32-line batches, each a list of (line, start misalignment)."""
    out = []
    for mis in (0, 5, 11):
        out.append([(_quoted(rng, 240), mis) for _ in range(32)])                     # every lane in the run
        b = [(_quoted(rng, 240), mis) for _ in range(32)]
        b[rng.randrange(32)] = (_word(rng, 240), mis)                                 # all but one lane
        out.append(b)
    for mis in (0, 7):
        for slot in range(16):  # one lane's exit byte at slot `slot` of chunk 4 (frame index 64 + slot)
            b = [(_quoted(rng, 250, close_at=246), mis) for _ in range(32)]
            j = (slot * 5 + mis) % 32
            b[j] = (_quoted(rng, 250, close_at=64 + slot - mis), mis)
            out.append(b)
    for _ in range(4):  # dead lanes next to live ones
        b = []
        for lane in range(32):
            n = rng.randint(150, 300)
            b.append((_dies(rng, n) if rng.random() < 0.4 else _quoted(rng, n), rng.randrange(16)))
        out.append(b)
    for _ in range(4):  # ragged lengths, every misalignment twice per warp
        mis = list(range(16)) * 2
        rng.shuffle(mis)
        b = []
        for lane in range(32):
            n = rng.choice((0, 1, 2, 15, 16, 17, 31, 33)) if rng.random() < 0.25 else rng.randint(18, 400)
            pick = rng.random()
            line = _quoted(rng, n) if pick < 0.6 else _word(rng, n) if pick < 0.8 else _dies(rng, n)
            b.append((line, mis[lane]))
        out.append(b)
    return out


def _arena(items):
    """Lines at 16-byte aligned slots plus their misalignment, with filler between them."""
    parts, off, ln, cur = [], [], [], 0
    for line, mis in items:
        start = ((cur + 15) & ~15) + mis
        parts.append(b"\x00" * (start - cur) + line)
        off.append(start)
        ln.append(len(line))
        cur = start + len(line)
    base = b"".join(parts) + b"\x00" * 32
    return np.frombuffer(base, np.uint8), np.array(off, np.uint32), np.array(ln, np.uint32)


def _items(order):
    """The batches once (natural order), or repeated to 4096 lines and more, so that the forced length-order pass
    runs (it needs that many events)."""
    batches = _batches(random.Random(20))
    items = [x for b in batches for x in b]
    if order == "1":
        rng = random.Random(21)
        while len(items) < 4096:
            items += [x for b in _batches(rng) for x in b]
    return items + items[:19]  # and a partial last batch


@pytest.fixture(scope="module", params=["0", "1"])
def case(request, lc):
    """(engine with the length-order pass off or forced on, buf, off, ln)."""
    mp = pytest.MonkeyPatch()
    mp.setenv("LC_B200_LENGTH_ORDER", request.param)
    e = lc.Engine(0)
    mp.undo()
    buf, off, ln = _arena(_items(request.param))
    yield e, buf, off, ln
    e.close()


def test_staged_kernel_warp_skip(lc, case):
    eng, buf, off, ln = case
    rx, orx = lc.Regex(SIMPLE), orc.Regex(SIMPLE)
    st, co, cl = eng.regex_parse(rx, buf, off, ln, 4)
    est, eco, ecl = orc.regex_parse_batch(orx, buf, off, ln, 4)
    assert (est == 0).any() and (est == 1).any()
    assert np.array_equal(st, est), np.nonzero(st != est)[0][:5]
    assert np.array_equal(co, eco[:, :rx.ngroups]) and np.array_equal(cl, ecl[:, :rx.ngroups])


def test_multi_kernel_warp_skip(lc, case):
    from loongcollector_b200 import synth
    eng, buf, off, ln = case
    pats, nkeys = [synth.NGINX_PATTERN, SIMPLE], [10, 4]
    rxs, orxs = [lc.Regex(p) for p in pats], [orc.Regex(p) for p in pats]
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
    assert (ewhich == 1).any() and (ewhich == 0xFF).any()
    assert np.array_equal(which, ewhich) and np.array_equal(status, est), np.nonzero(status != est)[0][:5]
    assert np.array_equal(co, eco) and np.array_equal(cl, ecl)
