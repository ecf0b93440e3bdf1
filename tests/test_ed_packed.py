"""A bit-exact model of ed_pack_kernel's packed column (edit_distance.cu), checked against a plain HW DP without a GPU.

Two HW queries of one target share one column of R = 32 W rows: A in rows 0 .. mA-1 with its last row in word WA, B in rows R-mB .. R-1,
and separator rows between them that match every byte and start at Pv = Mv = 0. The model follows the kernel word by word: the Peq
combine of build_pack_peq (B's words in its own class's HW layout placed at the top, words of separator rows only all ones, A's words from
the bottom with A's last word taking what lies above mA from B's side), the add with carry across the W words, the one-row shift with
carry, the SEP mask that clears bit mA & 31 of word WA in the new Pv and Mv, B's score read at bit 31 of the top word and A's through the
multiply by 2^(31 - s). Rows past a query's end hold garbage, as in the kernel, where the Peq build reads past the query."""
import numpy as np
import pytest

M32 = 0xFFFFFFFF
PACKS = ((3, 1), (5, 2))
ALPHA = b"ACGT"


def pack_fits(ma, mb, w, wa):
    return 32 * wa < ma <= 32 * wa + 31 and mb >= 1 and ma + mb < 32 * w


def _words(q, nw, c, garbage):
    """Match bits of q against the byte c in nw words, bit i = row i; rows past |q| take bits of `garbage`."""
    e = [0] * nw
    for r in range(32 * nw):
        bit = (q[r] == c) if r < len(q) else (garbage >> r) & 1
        e[r >> 5] |= int(bit) << (r & 31)
    return e


def _rows_to_top(e, p, vmask):
    for w in range(len(e) - 1, 0, -1):
        e[w] = ((e[w] << p) | (e[w - 1] >> (32 - p))) & M32 if p else e[w]
    e[0] = ((e[0] << p) & M32) | vmask
    return e


def _rows_in(w, lo, hi):
    def below(x):
        return 0 if x <= 0 else M32 if x >= 32 else (1 << x) - 1
    return below(hi - 32 * w) & ~below(lo - 32 * w) & M32


def pack_peq(qa, qb, w, wa, c, rng):
    """The W words of the packed Peq table for the byte c, as build_pack_peq stores them."""
    ma, mb = len(qa), len(qb)
    nb = (mb + 31) // 32
    col = [None] * w
    p = 32 * nb - mb
    col[w - nb:] = _rows_to_top(_words(qb, nb, c, int(rng.integers(0, 1 << 62)) << 40 | int(rng.integers(0, 1 << 40))), p, (1 << p) - 1)
    for x in range(wa, w - nb):
        col[x] = M32
    a = _words(qa, wa + 1, c, int(rng.integers(0, 1 << 62)) << 40 | int(rng.integers(0, 1 << 40)))
    low = ((2 << ((ma - 1) & 31)) - 1) & M32
    for x in range(wa):
        col[x] = a[x]
    col[wa] = (a[wa] & low) | (col[wa] & ~low & M32)
    return col


def packed_scores(qa, qb, t, w, wa, rng):
    """Per target column c = 1..|t|: (D_A[mA][c], D_B[mB][c]) from the packed column; asserts that the separator rows stay at
    Pv = Mv = 0 in every column."""
    ma, mb = len(qa), len(qb)
    assert pack_fits(ma, mb, w, wa)
    b0 = 32 * w - mb
    peq = {c: pack_peq(qa, qb, w, wa, c, rng) for c in set(t)}
    sepr = [_rows_in(x, ma, b0) for x in range(w)]
    pv = [~s & M32 for s in sepr]
    mv = [0] * w
    sep = 1 << (ma & 31)
    mula = 1 << (31 - ((ma - 1) & 31))
    sa, sb = ma, mb
    out = []
    for c in t:
        eq = peq[c]
        xv = [eq[x] | mv[x] for x in range(w)]
        tt = [eq[x] & pv[x] for x in range(w)]
        s, carry = [0] * w, 0
        for x in range(w):                                    # add.cc / addc chain
            v = tt[x] + pv[x] + carry
            s[x], carry = v & M32, v >> 32
        xh = [(s[x] ^ pv[x]) | eq[x] for x in range(w)]
        ph = [(mv[x] | ~(xh[x] | pv[x])) & M32 for x in range(w)]
        mh = [pv[x] & xh[x] for x in range(w)]
        sb += (ph[w - 1] >> 31) - (mh[w - 1] >> 31)           # two LEA.HI of the top word
        sa += (((ph[wa] * mula) & M32) >> 31) - (((mh[wa] * mula) & M32) >> 31)   # IMAD by 2^(31-s), then LEA.HI
        cp = cm = 0                                           # HW: the free top row shifts in 0
        for x in range(w):
            phs, mhs = ((ph[x] << 1) | cp) & M32, ((mh[x] << 1) | cm) & M32
            cp, cm = ph[x] >> 31, mh[x] >> 31
            pv[x] = (mhs | ~(xv[x] | phs)) & M32
            mv[x] = phs & xv[x]
            if x == wa:
                pv[x] &= ~sep & M32
                mv[x] &= ~sep & M32
        assert all((pv[x] | mv[x]) & sepr[x] == 0 for x in range(w)), "separator row left Pv = Mv = 0"
        out.append((sa, sb))
    return out


def hw_last_row(q, t):
    """D[m][c] for c = 1..|t| of the HW DP (free start in the target), byte equality."""
    m = len(q)
    col = np.arange(m + 1)
    res = []
    for c in t:
        new = np.empty_like(col)
        new[0] = 0
        for i in range(1, m + 1):
            new[i] = min(col[i - 1] + (q[i - 1] != c), col[i] + 1, new[i - 1] + 1)
        col = new
        res.append(int(col[m]))
    return res


def _check(qa, qb, t, w, wa, seed=0):
    got = packed_scores(qa, qb, t, w, wa, np.random.default_rng(seed))
    assert [g[0] for g in got] == hw_last_row(qa, t)
    assert [g[1] for g in got] == hw_last_row(qb, t)


def _rand(rng, n, alpha=ALPHA):
    return bytes(alpha[i] for i in rng.integers(0, len(alpha), size=n))


def _probe(rng, t, m):
    if m <= len(t) and rng.random() < 0.7:
        a0 = int(rng.integers(0, len(t) - m + 1))
        q = bytearray(t[a0:a0 + m])
        for i in np.nonzero(rng.random(m) < 0.05)[0]:
            q[i] = ALPHA[int(rng.integers(0, 4))]
        return bytes(q)
    return _rand(rng, m)


@pytest.mark.parametrize("w,wa", PACKS)
def test_random_pairs(w, wa):
    rng = np.random.default_rng(w)
    for _ in range(40):
        ma = int(rng.integers(32 * wa + 1, 32 * wa + 32))
        mb = int(rng.integers(1, 32 * w - ma))
        t = _rand(rng, int(rng.integers(1, 171)), b"ACGTNRacgt")
        _check(_probe(rng, t, ma), _probe(rng, t, mb), t, w, wa, seed=int(rng.integers(0, 1 << 30)))


@pytest.mark.parametrize("ma", [33, 63, 65, 95])
def test_a_at_the_ends_of_its_word(ma):
    w, wa = (3, 1) if ma < 64 else (5, 2)
    rng = np.random.default_rng(ma)
    for mb in (1, 2, 31, 32, 33, 32 * w - ma - 1):
        if mb >= 1 and pack_fits(ma, mb, w, wa):
            t = _rand(rng, 150)
            _check(_probe(rng, t, ma), _probe(rng, t, mb), t, w, wa, seed=mb)


@pytest.mark.parametrize("w,wa", PACKS)
def test_single_separator_row(w, wa):
    rng = np.random.default_rng(10 + w)
    for ma in (32 * wa + 1, 32 * wa + 16, 32 * wa + 31):
        mb = 32 * w - ma - 1                               # mA + mB + 1 = R
        assert pack_fits(ma, mb, w, wa) and not pack_fits(ma, mb + 1, w, wa)
        t = _rand(rng, 150)
        _check(_probe(rng, t, ma), _probe(rng, t, mb), t, w, wa, seed=ma)


@pytest.mark.parametrize("w,wa", PACKS)
def test_a_top_row_flips_every_column(w, wa):
    """A = (AC)* against (AC)*: A's last-row delta flips sign in every column, so the row above it takes a leak of the opposite kind
    every column and the SEP mask must clear it each time."""
    ma = 32 * wa + 17
    qa = (b"AC" * 64)[:ma]
    t = b"AC" * 75
    d = np.diff(hw_last_row(qa, t)[ma:])
    assert len(d) > 50 and np.all(d[1:] == -d[:-1]) and np.all(d != 0)
    for mb in (1, 32 * w - ma - 1):
        _check(qa, _rand(np.random.default_rng(mb), mb), t, w, wa, seed=mb)


def test_pack_bounds():
    assert pack_fits(33, 62, 3, 1) and not pack_fits(33, 63, 3, 1) and not pack_fits(64, 1, 3, 1) and not pack_fits(32, 1, 3, 1)
    assert pack_fits(95, 64, 5, 2) and not pack_fits(95, 65, 5, 2) and not pack_fits(96, 1, 5, 2) and not pack_fits(64, 1, 5, 2)
    # the benchmark's probe pairs (two probes of one length, 26-80 bp) pack at 33-47 and 65-79 bp
    fits = {m for m in range(26, 81) for w, wa in PACKS if pack_fits(m, m, w, wa)}
    assert fits == set(range(33, 48)) | set(range(65, 80))
