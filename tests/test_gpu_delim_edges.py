"""GPU tier: the delimiter kernels at the shapes where their own code (not the shared state machine) can go wrong.

Every length 0..300 at every 16-byte alignment, records of up to 1 MiB in one warp batch with short ones, leading and
trailing blank runs that cross the 32-byte steps and 128-byte stages of delim_tiled_kernel, all four kernel paths of
launch_delim, configurations at their edges and the column tap.  Every call goes through lc_delim_parse_tap_dev on
output tables that are filled with a poison word and followed by guard words, so a kernel that leaves a column unwritten
or writes past row n - 1 fails; every row is compared with oracle.delim_parse_batch on the same bytes."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as orc  # noqa: E402  (checker only)

HERE = os.path.dirname(os.path.abspath(__file__))
POISON = 0xA5A5A5A5
GUARD = 67  # poison words behind every table

# (separator, quote): the quote state machine (tiled kernel for MF <= 32), the blank separator / blank quote that
# interact with the trim, and the SplitString path (multi-byte separator, or quote == separator)
SEPQ = [(b",", '"'), (b"\t", '"'), (b" ", '"'), (b",", " "), (b"|", "'"), (b",", ","), (b"@@", '"'), (b"||a", '"'),
        (b"abcd", '"')]
# <= 32: tiled kernel (quote machine) / delim_kernel<true> (SplitString); > 32: delim_kernel<false>
MFS = (1, 3, 11, 32, 33, 64)
NKEYS = (0, 1, 4, 40)
MODES = ((True, True), (False, True), (False, False))  # (extend, allow_short)
BOUNDS = (16, 32, 128, 256)  # 16-byte chunk, 32-byte step, 128-byte stage, second stage
ORDINARY = b"abcxyz019-.:/_\xc3\xa9\xff\x80"


def _id(sq):
    return "%s-%s" % (sq[0].decode().replace("\t", "tab").replace(" ", "blank"), {" ": "blank"}.get(sq[1], sq[1]))


@pytest.fixture(scope="module")
def eng():
    import loongcollector_b200 as lc
    e = lc.Engine(0)
    yield e
    e.close()


# ------------------------------------------------------------------------------------------- records
class Records:
    """Delimiter records of an exact length for one (separator, quote) pair."""

    def __init__(self, rng, sep, quote):
        self.rng, self.sep, self.q = rng, sep, quote.encode()
        alpha = bytes(c for c in ORDINARY if c not in sep and c != self.q[0])
        # random slices of two fixed random strings: one random draw per run of bytes instead of one per byte
        self.pool = bytes(rng.choices(alpha, k=1 << 16))
        self.blank_pool = bytes(rng.choices(b" \r", k=1 << 16))

    def _slice(self, pool, n):
        if n > len(pool):
            pool *= n // len(pool) + 1
        s = self.rng.randrange(len(pool) - n + 1)
        return pool[s:s + n]

    def plain(self, n):  # ordinary bytes: no separator, quote or blank
        return self._slice(self.pool, n)

    def body(self, n):  # inside a quoted column: ordinary bytes, separators, doubled quotes
        out = bytearray()
        while len(out) < n:
            r = self.rng.random()
            if r < 0.12 and n - len(out) >= 2:
                out += self.q * 2
            elif r < 0.3 and n - len(out) >= len(self.sep):
                out += self.sep
            else:
                out += self.plain(min(n - len(out), self.rng.randint(1, 40)))
        return bytes(out)

    def quoted(self, n):
        return self.q + self.body(n - 2) + self.q

    def cell(self, n):
        return self.quoted(n) if n >= 2 and self.rng.random() < 0.4 else self.plain(n)

    def wf(self, n):
        """well-formed: columns joined by the separator, exactly n bytes"""
        d = len(self.sep)
        k = self.rng.randint(1, max(1, min(n // (d + 2), self.rng.choice((3, 12, 90)))))
        room = n - (k - 1) * d
        cuts = sorted(self.rng.randint(0, room) for _ in range(k - 1))
        return self.sep.join(self.cell(b - a) for a, b in zip([0] + cuts, cuts + [room]))

    def head(self, a):  # a bytes that end a column, so that a new column starts at offset a
        d = len(self.sep)
        return b"" if a == 0 else (self.wf(a - d) + self.sep if a >= d else None)

    def tail(self, m):  # m bytes behind a column that ends here
        d = len(self.sep)
        return b"" if m == 0 else (self.sep + self.wf(m - d) if m >= d else None)

    def decisive(self, L, p, kind):
        """a record of length L whose decisive pair of bytes sits at offsets p | p + 1 (None: does not fit)"""
        rng, q = self.rng, self.q
        if p < 0 or p + 1 >= L:
            return None
        parts = None
        if kind == "sep|open":  # a column opens with a quote at p + 1
            b = rng.randint(p + 2, L - 1) if p + 2 <= L - 1 else None
            if b is not None:
                parts = [self.head(p + 1), self.quoted(b - p), self.tail(L - 1 - b)]
        elif kind == "open|x":  # opening quote at p, its first content byte at p + 1
            b = rng.randint(p + 2, L - 1) if p + 2 <= L - 1 else None
            if b is not None:
                parts = [self.head(p), self.quoted(b - p + 1), self.tail(L - 1 - b)]
        elif kind == "close|sep":  # closing quote at p, separator at p + 1
            if p >= 1:
                a = rng.randint(max(0, p - 40), p - 1)
                parts = [self.head(a), self.quoted(p - a + 1), self.tail(L - 1 - p)]
        elif kind == "x|close":  # last content byte at p, closing quote at p + 1
            if p >= 1:
                a = rng.randint(max(0, p - 40), p - 1)
                parts = [self.head(a), self.quoted(p - a + 2), self.tail(L - 2 - p)]
        elif kind == "dq":  # the two halves of a doubled quote at p | p + 1
            if p >= 1 and p + 2 <= L - 1:
                a = rng.randint(max(0, p - 40), p - 1)
                b = rng.randint(p + 2, min(L - 1, p + 40))
                cell = q + self.body(p - a - 1) + q * 2 + self.body(b - p - 2) + q
                parts = [self.head(a), cell, self.tail(L - 1 - b)]
        elif kind == "data|quote":  # unquoted data at p, an erroneous quote at p + 1
            a = rng.randint(max(0, p - 40), p)
            parts = [self.head(a), self.plain(p - a + 1), q, self.wf(L - p - 2)]
        elif kind == "quote@p":  # unquoted data in front of p, an erroneous quote at p
            if p >= 1:
                a = rng.randint(max(0, p - 40), p - 1)
                parts = [self.head(a), self.plain(p - a), q, self.wf(L - p - 1)]
        elif kind == "close|byte":  # closing quote at p, an ordinary byte at p + 1
            if p >= 1:
                a = rng.randint(max(0, p - 40), p - 1)
                parts = [self.head(a), self.quoted(p - a + 1), self.plain(1), self.wf(L - p - 2)]
        elif kind == "unterminated":  # a quote opens at p + 1 and is never closed
            parts = [self.head(p + 1), q, self.body(L - p - 2)]
        else:
            raise AssertionError(kind)
        if parts is None or any(x is None for x in parts):
            return None
        rec = b"".join(parts)
        assert len(rec) == L, (kind, L, p, len(rec))
        return rec

    def blanks(self, n):  # trailing run: ' ' and '\r' mixed
        return self._slice(self.blank_pool, n)


WELL = ("sep|open", "open|x", "close|sep", "x|close", "dq")
BAD = ("data|quote", "quote@p", "close|byte", "unterminated")


def _boundary_record(R, L, mis, j, kinds):
    """kinds[j]-style record with its decisive pair on a step / stage boundary: in the 16-byte frame the kernels read
    (every other record) or at the line offset itself"""
    for t in range(len(BOUNDS) * len(kinds)):
        B = BOUNDS[(j + t) % len(BOUNDS)]
        p = B - 1 - (mis if (j // 2) % 2 == 0 else 0)
        rec = R.decisive(L, p, kinds[(j + t // len(BOUNDS)) % len(kinds)])
        if rec is not None:
            return rec
    return None


def _mixed_record(R, L, mis, j):
    """item j of the rotation well-formed / malformed / blank-padded, exactly L bytes"""
    kind = j % 3
    if kind == 0:
        rec = _boundary_record(R, L, mis, j // 3, WELL)
        return rec if rec is not None else R.wf(L)
    if kind == 1:
        rec = _boundary_record(R, L, mis, j // 3, BAD)
        if rec is not None:
            return rec
        return (R.q + R.plain(L - 1)) if L else b""
    # blank-padded: the first non-blank byte on a boundary (or anywhere), trailing ' ' / '\r' run
    B = BOUNDS[(j // 3) % len(BOUNDS)] - mis - (j // 12) % 2
    lead = B if 0 <= B <= L and j % 2 else R.rng.randint(0, L)
    trail = R.rng.randint(0, L - lead)
    return b" " * lead + R.wf(L - lead - trail) + R.blanks(trail)


def _arena(records, aligns, shift, sep, quote):
    """records laid out one behind the other, record k starting at frame offset aligns[k] (mod 16) of an arena that
    begins `shift` bytes into a 16-byte aligned allocation.  Every gap (at least one byte) and the tail rotate through
    the separator, the quote, ' ' and '\\r', so any read outside [off, off + len) changes a result."""
    fill = bytes([sep[0], ord(quote), 0x20, 0x0D])
    pieces, offs, lens = [], [], []
    at = 0
    for k, rec in enumerate(records):
        pad = (aligns[k] - (shift + at)) % 16 or 16
        pieces.append(bytes(fill[(k + t) % 4] for t in range(pad)))
        at += pad
        pieces.append(rec)
        offs.append(at)
        lens.append(len(rec))
        at += len(rec)
    pieces.append(bytes(fill[t % 4] for t in range(64)))
    return np.frombuffer(b"".join(pieces), np.uint8), np.array(offs, np.uint32), np.array(lens, np.uint32)


# ------------------------------------------------------------------------------------------- device runner
class Dev:
    """An arena and its line table in HBM; parse() runs lc_delim_parse_tap_dev on poisoned, guarded tables."""

    def __init__(self, base, off, ln, shift):
        import torch
        self.torch = torch
        self.dev = torch.device("cuda", 0)
        self.base, self.off, self.ln, self.shift = base, off, ln, shift
        self.n = off.size
        t = torch.full((base.size + shift + 64,), 0x20, dtype=torch.uint8, device=self.dev)
        t[shift:shift + base.size] = torch.from_numpy(base.copy()).to(self.dev)
        self.d_base = t
        self.d_off = torch.from_numpy(off.view(np.int32).copy()).to(self.dev)
        self.d_len = torch.from_numpy(ln.view(np.int32).copy()).to(self.dev)

    def _table(self, count, word_shift, itemsize=4):
        torch = self.torch
        if itemsize == 1:
            return torch.full((word_shift + count + GUARD,), 0xA5, dtype=torch.uint8, device=self.dev)
        return torch.full((word_shift + count + GUARD,), POISON - (1 << 32), dtype=torch.int32, device=self.dev)

    def parse(self, eng, sep, quote, nkeys, extend, allow_short, mf, word_shift=0, tap_col=None):
        n, ws = self.n, word_shift
        tabs = [self._table(n, ws, 1), self._table(n, ws)] + [self._table(n * mf, ws) for _ in range(3)]
        taps = [self._table(n, ws), self._table(n, ws)] if tap_col is not None else [None, None]
        ptr = [t.data_ptr() + ws * t.element_size() for t in tabs]
        tptr = [t.data_ptr() + ws * 4 if t is not None else None for t in taps]
        eng.delim_parse_dev(self.d_base.data_ptr() + self.shift, self.base.size, self.d_off.data_ptr(),
                            self.d_len.data_ptr(), n, sep, ord(quote), nkeys, extend, allow_short, mf, *ptr,
                            tap_col=tap_col, d_tap_off=tptr[0], d_tap_len=tptr[1])
        eng.sync()
        out = []
        for t, count in zip(tabs + [x for x in taps if x is not None], [n, n] + [n * mf] * 3 + [n, n]):
            h = t.cpu().numpy()
            h = h if h.dtype == np.uint8 else h.view(np.uint32)
            poison = 0xA5 if h.dtype == np.uint8 else POISON
            assert np.all(h[:ws] == poison) and np.all(h[ws + count:] == poison), \
                ("write outside the table", count, np.nonzero(h[ws + count:] != poison)[0][:4])
            out.append(h[ws:ws + count])
        st, nf = out[0], out[1]
        fo, fl, fd = (x.reshape(n, mf) for x in out[2:5])
        return (st, nf, fo, fl, fd) + tuple(out[5:])

    def check(self, eng, sep, quote, nkeys, extend, allow_short, mf, word_shift=0, tap_col=None):
        """every row against the oracle; returns the oracle's status column"""
        got = self.parse(eng, sep, quote, nkeys, extend, allow_short, mf, word_shift, tap_col)
        want = orc.delim_parse_batch(self.base, self.off, self.ln, sep, ord(quote), nkeys, extend, allow_short, mf)
        what = (sep, quote, nkeys, extend, allow_short, mf, self.shift, word_shift, tap_col)
        for g, w, name in zip(got, want, ("status", "nfields", "f_off", "f_len", "f_dq")):
            bad = np.nonzero((g != w).reshape(self.n, -1).any(axis=1))[0]
            if bad.size:
                i = int(bad[0])
                o, L = int(self.off[i]), int(self.ln[i])
                raise AssertionError(
                    "%s differs in %d rows; first: row %d, len %d, frame offset %d, %r; got %s, want %s %r"
                    % (name, bad.size, i, L, (o + self.shift) % 16, bytes(self.base[o:o + min(L, 80)]),
                       g[i] if g.ndim == 1 else g[i].tolist()[:12], w[i] if w.ndim == 1 else w[i].tolist()[:12], what))
        if tap_col is not None:
            t_off, t_len = got[5], got[6]
            assert np.array_equal(t_off, want[2][:, tap_col]) and np.array_equal(t_len, want[3][:, tap_col]), \
                ("tap",) + what
            empty = (want[0] == 1) | (want[0] == 2) | (want[1] <= tap_col)  # failed, blank, too few columns
            assert not np.any(t_off[empty]) and not np.any(t_len[empty]), ("tap",) + what
        return want[0]


def _verdicts(st, nkeys, sep, quote, what):
    """accepted and rejected records both occur (for nkeys == 0 no record is accepted: failed and blank then)"""
    if nkeys == 0:
        assert np.any(st == 1) and np.any(st == 2), what
        return
    assert np.any(st == 0) and np.any(st != 0), what
    if len(sep) == 1 and ord(quote) != sep[0]:
        assert np.any(st == 1), what  # malformed records rejected by the state machine


def _calls():
    """(max_fields, nkeys, extend, allow_short) for one arena: every MF with every nkeys, the three modes rotating"""
    out = []
    for a, mf in enumerate(MFS):
        for b, nk in enumerate(NKEYS):
            out.append((mf, nk) + MODES[(a + b) % 3])
    return out


def _tap(mf, j):
    col = (None, 0, 3, mf - 1)[j % 4]
    return col if col is None or col < mf else mf - 1


# ------------------------------------------------------------------------------------------- 1. lengths x alignments
@pytest.mark.parametrize("sep,quote", SEPQ, ids=[_id(x) for x in SEPQ])
def test_every_length_at_every_alignment(eng, sep, quote):
    """Lengths 0..300 (the 16-byte chunk, the 32-byte step and both stage boundaries) at every frame offset, base
    shifted by 0 and 7 bytes; well-formed, malformed and blank-padded records with the decisive bytes on the boundary
    bytes; long and short lines in random order, so that stale tile slots hold the filler bytes."""
    rng = random.Random("%r%s" % (sep, quote))
    R = Records(rng, sep, quote)
    pairs = [(L, a) for L in range(301) for a in range(16)]
    rng.shuffle(pairs)
    records = [_mixed_record(R, L, a, j) for j, (L, a) in enumerate(pairs)]
    for shift in (0, 7):  # (a record's frame offset does not depend on the shift: same records, other gaps)
        base, off, ln = _arena(records, [a for _, a in pairs], shift, sep, quote)
        assert np.array_equal(ln, [L for L, _ in pairs])
        assert np.array_equal((off + shift) % 16, [a for _, a in pairs])
        d = Dev(base, off, ln, shift)
        for j, (mf, nk, ext, short) in enumerate(_calls()):
            st = d.check(eng, sep, quote, nk, ext, short, mf, word_shift=j % 2, tap_col=_tap(mf, j))
            _verdicts(st, nk, sep, quote, (sep, quote, shift, mf, nk, ext, short))


# ------------------------------------------------------------------------------------------- 3. blank runs
def _blank_records(R, sep):
    rng, q = R.rng, R.q
    recs = []
    for n in range(301):
        # leading ' ' run of n bytes in front of a short record (the first non-blank byte n bytes in), and in front of
        # a record of 0..300 bytes behind which a trailing run of ' ' / '\r' follows
        recs.append(b" " * n + R.wf(rng.randint(1, 12)))
        recs.append(b" " * n + R.wf(rng.randint(0, 300)) + R.blanks(rng.randint(0, 300)))
        # trailing run of n mixed ' ' / '\r' bytes
        recs.append(R.wf(rng.randint(1, 300)) + R.blanks(n))
        recs.append(R.plain(1) + R.blanks(n))
        # all blank
        recs.append(b" " * n)
        recs.append(R.blanks(n))
        # the only non-blank byte at offset n (an ordinary byte, a quote, the separator's first byte), and at the end
        # of a line of 300
        for c in (R.plain(1), q, sep[:1]):
            recs.append(b" " * n + c + R.blanks(rng.randint(0, 300 - n)))
        if n < 300:
            recs.append(R.blanks(300)[:n] + R.plain(1) + R.blanks(299 - n))
    # a '\r' that leads or sits inside the record is not trimmed
    for n in (1, 2, 15, 16, 17, 31, 32, 33, 127, 128, 129, 255, 256, 257):
        recs.append(b"\r" * n + R.wf(rng.randint(0, 40)))
        recs.append(b" " * n + b"\r" + R.wf(rng.randint(0, 40)) + R.blanks(n))
        recs.append(R.wf(n) + b"\r" + R.wf(rng.randint(0, 40)) + b" \r" * (n // 2))
        recs.append(b"\r" + b" " * n + b"\r")
    return recs


@pytest.mark.parametrize("sep,quote", SEPQ, ids=[_id(x) for x in SEPQ])
def test_blank_runs(eng, sep, quote):
    """Leading ' ' runs and trailing ' ' / '\\r' runs of 0..300 bytes, all-blank lines of every length 0..300, lines
    whose only non-blank byte sits at every offset, a '\\r' at the start or inside (not trimmed there)."""
    rng = random.Random("blank%r%s" % (sep, quote))
    records = _blank_records(Records(rng, sep, quote), sep)
    rng.shuffle(records)
    for shift in (0, 7):
        base, off, ln = _arena(records, [k % 16 for k in range(len(records))], shift, sep, quote)
        d = Dev(base, off, ln, shift)
        for j, (mf, nk, ext, short) in enumerate(_calls()):
            if (j + shift) % 2:
                continue  # half of the calls per shift: each shift sees every MF and every nkeys
            st = d.check(eng, sep, quote, nk, ext, short, mf, word_shift=(j // 2) % 2, tap_col=_tap(mf, j // 2))
            assert np.any(st == 2), (sep, quote, mf, nk)
            if nk:
                assert np.any(st == 0), (sep, quote, mf, nk)


# ------------------------------------------------------------------------------------------- 2. long records
LONG = (4095, 4096, 4097, 65535, 65536, 70001, 1 << 20)


@pytest.mark.parametrize("sep,quote", [(b",", '"'), (b"\t", "'"), (b" ", '"'), (b"@@", '"')],
                         ids=["comma", "tab", "blank", "atat"])
def test_long_records_in_warp_batches_with_short_ones(eng, sep, quote):
    """Records of 4 KiB .. 1 MiB -- well-formed with quoted columns of several KB that span many stages, malformed
    late in the record, blank-padded by KB-long runs -- each in a 32-line batch with 31 short lines, so one lane sets
    the batch's stage count for the others."""
    rng = random.Random("long%r" % sep)
    R = Records(rng, sep, quote)
    longs = []
    for L in LONG:
        # well-formed: six columns, the quoted ones several KB long
        w = L // 6 - len(sep)
        rec = sep.join(R.quoted(w) if c % 2 else R.plain(w) for c in range(5)) + sep
        longs.append(rec + R.wf(L - len(rec)))
        # malformed only late in the record: a byte behind a closing quote and an erroneous quote on a stage boundary,
        # a quote that opens a third in and is never closed, an erroneous quote as the last byte
        p = ((L - 300) & ~127) - 1
        longs += [R.decisive(L, p, "close|byte"), R.decisive(L, p, "data|quote"),
                  R.decisive(L, L // 3, "unterminated"), R.plain(L - 1) + R.q]
        # blank-padded: KB-long leading and trailing runs
        lead, trail = L // 3 + 5, L // 4 + 3
        longs.append(b" " * lead + R.wf(L - lead - trail) + R.blanks(trail))
    rng.shuffle(longs)
    records = []
    for b, rec in enumerate(longs):
        block = [_mixed_record(R, rng.randint(0, 60), 0, j) for j in range(31)]
        block.insert((b * 7) % 32, rec)  # one long line per batch of 32, at varying lanes
        records += block
    base, off, ln = _arena(records, [rng.randrange(16) for _ in records], 3, sep, quote)
    assert sorted(int(x) for x in ln if x >= 4095) == sorted(len(r) for r in longs)
    d = Dev(base, off, ln, 3)
    for j, (mf, nk, ext, short) in enumerate([(11, 4, True, True), (3, 40, False, True), (33, 4, False, False),
                                              (64, 40, True, True), (32, 1, False, False)]):
        st = d.check(eng, sep, quote, nk, ext, short, mf, word_shift=j % 2, tap_col=_tap(mf, j + 1))
        long_st = st[ln >= 4095]
        assert np.any(long_st == 0), (sep, mf, nk)
        if len(sep) == 1:
            assert np.any(long_st == 1), (sep, mf, nk)


# ------------------------------------------------------------------------------------------- 6. tables
@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 32 * 97 + 1])
def test_output_tables_of_partly_full_batches(eng, n):
    """The last batch of 32 is partly full; nothing may be written behind row n - 1 (guard words), no cell may keep
    its poison; table pointers one word off their 16-byte alignment take the scalar copy-out."""
    rng = random.Random(n)
    for sep, quote, mf in ((b",", '"', 11), (b"|", "'", 32), (b",", '"', 33), (b"@@", '"', 11), (b",", ",", 64),
                           (b"\t", '"', 1)):
        R = Records(rng, sep, quote)
        records = [_mixed_record(R, rng.choice((0, 5, 40, 130, 300)), 0, j) for j in range(n)]
        base, off, ln = _arena(records, [rng.randrange(16) for _ in records], 0, sep, quote)
        d = Dev(base, off, ln, 0)
        for ws in (0, 1):
            d.check(eng, sep, quote, 4, True, True, mf, word_shift=ws, tap_col=mf - 1)
            d.check(eng, sep, quote, 40, False, False, mf, word_shift=ws)


# ------------------------------------------------------------------------------------------- 7. tap
def test_tap_column_outside_the_table_is_rejected(eng):
    import loongcollector_b200 as lc
    rng = random.Random(5)
    R = Records(rng, b",", '"')
    records = [R.wf(rng.randint(0, 80)) for _ in range(100)]
    base, off, ln = _arena(records, [0] * 100, 0, b",", '"')
    d = Dev(base, off, ln, 0)
    for mf, col in ((11, 11), (11, 12), (33, 40), (1, 1)):
        with pytest.raises(lc.LcError) as ei:
            d.parse(eng, b",", '"', 4, True, True, mf, tap_col=col)
        assert ei.value.code == lc.capi.LC_ERR_INVALID_ARG


# ------------------------------------------------------------------------------------------- 4. knobs
@pytest.mark.timeout(300)
@pytest.mark.parametrize("knob", ["LC_B200_DELIM_NO_TILE", "LC_B200_DELIM_DIRECT"])
def test_delimiter_knobs_agree(knob):
    """The knobs are read once per process: the length / alignment and blank-run tests run again in a fresh interpreter
    with the knob set (NO_TILE: delim_kernel<true> runs the quote machine; DIRECT: delim_kernel<false> for every MF)."""
    env = dict(os.environ, **{knob: "1"})
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", __file__, "-k",
                        "every_length or blank_runs"], env=env, capture_output=True, text=True,
                       timeout=280, cwd=os.path.dirname(HERE))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
