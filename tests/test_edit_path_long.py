"""Edit paths and distances where the device code has the most room to go wrong: sequences that share arena bytes, aligned target slices from
4 kb up to the 16384-column limit (segment classes 9-11 and status 2), deep Hirschberg recursion, and multi-stripe edit distances.

Every path is compared with the reference's edlib (compiled verbatim) op for op, and replayed against the sequences on its own: the ops must
consume exactly q and t[start..end], use op 0 only on equal bytes and op 3 only on unequal ones, and contain dist edits."""
import os
import subprocess
import sys

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALPHA = np.frombuffer(b"ACGT", np.uint8)
AMB = np.frombuffer(b"MRWBSYDKEF-N", np.uint8)
IUPAC_EQ = b"MAMCRARGWAWTBAB-SCSGYCYTDCD-KGKTEGE-FTF-"  # the 20 pairs of src/assemble.h:425
EQS = pytest.mark.parametrize("eq", [b"", IUPAC_EQ], ids=["plain", "iupac"])
SLICE_LIMIT = 16384                                     # widest aligned target slice dgpu_edit_path traces (status 2 beyond)
SLICES = [4096, 4097, 6000, 8192, 8193, 12000, 16383, 16384]


def _rand(rng, n):
    return ALPHA[rng.integers(0, 4, size=n)]


def _sprinkle(rng, t, frac=0.04):
    """IUPAC codes and gaps in place of a few bases, as in a gapped consensus."""
    t = t.copy()
    k = max(1, int(len(t) * frac))
    t[rng.integers(0, len(t), size=k)] = AMB[rng.integers(0, len(AMB), size=k)]
    return t


def _noisy(rng, s, rate, flank=32):
    """Substitutions and indels inside s; the flanks stay exact so that the aligned slice keeps the length of s."""
    mid = synth.mutate_fast(rng, s[flank:len(s) - flank], sub=0.6 * rate, ins=0.2 * rate, dele=0.2 * rate)
    return np.concatenate([s[:flank], mid, s[len(s) - flank:]])


def _batch(arena, jobs):
    j = np.array(jobs, np.int64).reshape(-1, 4)
    u = lambda c: np.ascontiguousarray(j[:, c].astype(np.uint32))
    return dict(seqs=np.ascontiguousarray(arena, np.uint8), q_off=u(0), q_len=u(1), t_off=u(2), t_len=u(3))


def _packed(seqs):
    arena, off, ln = synth.pack(seqs)
    return dict(seqs=arena, q_off=off[0::2].copy(), q_len=ln[0::2].copy(), t_off=off[1::2].copy(), t_len=ln[1::2].copy())


def _seq(b, i, which):
    o, n = int(b[which + "_off"][i]), int(b[which + "_len"][i])
    return b["seqs"][o:o + n].tobytes()


def _eq_table(eq):
    tab = np.eye(256, dtype=bool)
    for i in range(0, len(eq), 2):
        tab[eq[i], eq[i + 1]] = tab[eq[i + 1], eq[i]] = True
    return tab


def _replay(q, t, d, s, e, ops, eq):
    """The path on its own: a script from q to t[s..e] with d edits, matches exactly on equal bytes (under the pairs)."""
    o = np.frombuffer(ops, np.uint8)
    assert o.size == 0 or o.max() <= 3
    qa, ta = np.frombuffer(q, np.uint8), np.frombuffer(t, np.uint8)
    assert int((o != 2).sum()) == len(q), "ops do not consume the query"
    assert int((o != 1).sum()) == e - s + 1, "ops do not consume t[start..end]"
    assert int((o != 0).sum()) == d, "edits differ from the distance"
    diag = (o == 0) | (o == 3)
    qi = np.cumsum(o != 2)[diag] - 1
    tj = s + np.cumsum(o != 1)[diag] - 1
    same = _eq_table(eq)[qa[qi], ta[tj]]
    assert np.array_equal(o[diag] == 0, same), "a match op on unequal bytes or a mismatch op on equal bytes"


def _check_paths(ctx, ref, b, mode, eq, status=None):
    """Device paths vs the reference's edlib. status: expected status per job (default all 0); a job with status 2 must still carry the
    reference's distance and locations, and no ops. Returns the reference's (dist, end, start) per job."""
    d, st, en, ops, stat = ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], mode, eq=eq)
    n = len(d)
    want = np.zeros(n, np.uint32) if status is None else np.asarray(status, np.uint32)
    out, bad = [], []
    for i in range(n):
        q, t = _seq(b, i, "q"), _seq(b, i, "t")
        rd, re, rs, rops = po.edit_distance(ref, q, t, -1, mode, task=1 if want[i] == 2 else 2, eq=eq)
        if (d[i], st[i], en[i], stat[i]) != (rd, rs, re, want[i]) or ops[i] != (b"" if want[i] == 2 else rops):
            # every wrong job with what it returned: (job, |q|, |t|, status, dist, start, end, ops length) vs the reference's
            bad.append((i, len(q), len(t), int(stat[i]), int(d[i]), int(st[i]), int(en[i]), len(ops[i]), "ref", int(want[i]), rd, rs, re, len(rops)))
        out.append((rd, re, rs))
    assert not bad, (mode, bad[:6])
    for i in range(n):
        if want[i] == 0:
            _replay(_seq(b, i, "q"), _seq(b, i, "t"), int(d[i]), int(st[i]), int(en[i]), ops[i], eq)
    return out


# ---------------------------------------------------------------------------------------------------------------------------------------
# 1. sequences that share arena bytes

def _shared_arena(eq, seed=515):
    """A 50 kb contig followed by reads drawn from it; jobs point anywhere into it, sharing bytes in every way the ABI allows."""
    rng = np.random.default_rng(seed)
    C = 50_000
    contig = _rand(rng, C)
    if eq:
        contig = _sprinkle(rng, contig)
    jobs, reads = [], []
    # query inside its target (the last one: the same bytes)
    for tl, a, ql in ((120, 40, 30), (700, 200, 300), (5000, 1700, 1500), (2600, 0, 900), (64, 0, 64)):
        o = int(rng.integers(0, C - tl))
        jobs.append((o + a, ql, o, tl))
    # query and target at the same offsets, the same length
    for L in (50, 129, 2100):
        o = int(rng.integers(0, C - L))
        jobs.append((o, L, o, L))
    # query overlapping the target's start, then its end
    for tl, ov, ql in ((300, 30, 80), (3000, 400, 900)):
        o = int(rng.integers(2000, C - tl - 2000))
        jobs.append((o - (ql - ov), ql, o, tl))
        jobs.append((o + tl - ov, ql, o, tl))
    # targets: overlapping windows of the contig at different offsets; queries: reads drawn from them (packed after the contig)
    wins = []
    for w in range(6):
        o, tl = 10_000 + 1500 * w, int(rng.integers(2500, 4500))
        a, ql = int(rng.integers(0, tl // 3)), int(rng.integers(tl // 3, 2 * tl // 3))
        reads.append(synth.mutate_fast(rng, contig[o + a:o + a + ql], sub=0.03, ins=0.01, dele=0.01))
        wins.append((o, tl))
    roff = C + np.concatenate([[0], np.cumsum([len(r) for r in reads])[:-1]])
    for w, (o, tl) in enumerate(wins):
        jobs.append((int(roff[w]), len(reads[w]), o, tl))
    # the query of one job is the target of another: window w against window w + 1, and a short read against window w's first bytes
    for w in range(len(wins) - 1):
        jobs.append((wins[w][0], wins[w][1], wins[w + 1][0], wins[w + 1][1]))
        jobs.append((wins[w][0] + 100, 100, wins[w][0], 600))
    return _batch(np.concatenate([contig] + reads), jobs)


@pytest.mark.gpu
@EQS
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_path_shared_arena_bytes(ctx, ref, mode, eq):
    """Queries inside, equal to or overlapping their targets, targets that are overlapping windows of one contig, and a query that is the
    target of another job: each job's path is the one of its own two sequences (the HW start pass reverses every job into private bytes)."""
    _check_paths(ctx, ref, _shared_arena(eq), mode, eq)


@pytest.mark.gpu
@EQS
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_distance_shared_arena_bytes(ctx, oracle, mode, eq):
    """The same layouts through dgpu_edit_distance (queries of <= 128 and of more bases), with end locations, k unbounded, below, at and
    above the distance. Sequences with IUPAC bytes are compared byte for byte here."""
    b = _shared_arena(eq)
    args = (b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"])
    od, oe = po.edit_distance_batch(oracle, *args, None, mode, threads=os.cpu_count() or 1, want_end=True)
    gd, ge = ctx.edit_distance(*args, None, mode, want_end=True)
    assert np.array_equal(gd, od) and np.array_equal(ge, oe)
    assert (b["q_len"] <= 128).sum() >= 4 and (b["q_len"] > 128).sum() >= 4
    for dk in (-1, 0, 1):
        k = np.maximum(od + dk, 0).astype(np.int32)
        od2, oe2 = po.edit_distance_batch(oracle, *args, k, mode, threads=os.cpu_count() or 1, want_end=True)
        gd2, ge2 = ctx.edit_distance(*args, k, mode, want_end=True)
        assert np.array_equal(gd2, od2), (dk, np.nonzero(gd2 != od2)[0][:8])
        assert np.array_equal(ge2, oe2), (dk, np.nonzero(ge2 != oe2)[0][:8])


@pytest.mark.gpu
def test_path_hw_many_jobs_on_one_window(ctx, ref):
    """30000 HW jobs of eight reads against one 40 kb window. The start pass reverses each job's two sequences into bytes of its own, in
    runs of at most 1 GiB (1.2 GB here: two runs); every job must give the path of its own pair, on both sides of the run boundary."""
    rng = np.random.default_rng(818)
    T, N = 40_000, 30_000
    t = _rand(rng, T)
    reads = []
    for _ in range(8):
        a, L = int(rng.integers(0, T - 300)), int(rng.integers(100, 300))
        reads.append(synth.mutate_fast(rng, t[a:a + L], sub=0.03, ins=0.01, dele=0.01))
    roff = T + np.concatenate([[0], np.cumsum([len(r) for r in reads])[:-1]])
    arena = np.concatenate([t] + reads)
    which = rng.integers(0, 8, size=N)
    assert (T + min(len(r) for r in reads)) * N > 1 << 30
    refs = [po.edit_distance(ref, r.tobytes(), t.tobytes(), -1, 2, task=2) for r in reads]   # (dist, end, start, ops)
    b = _batch(arena, [(int(roff[w]), len(reads[w]), 0, T) for w in which])
    d, st, en, ops, stat = ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], 2)
    assert not stat.any()
    exp = np.array([refs[w][:3] for w in which])
    bad = np.nonzero((d != exp[:, 0]) | (en != exp[:, 1]) | (st != exp[:, 2]))[0]
    assert bad.size == 0, (bad.size, bad[:8])
    assert all(ops[i] == refs[w][3] for i, w in enumerate(which))


@pytest.mark.gpu
def test_long_needle_shared_arena_bytes(ctx, ref):
    """longNeedle with the consensus a sub-window of its own reference window (and overlapping its ends)."""
    rng = np.random.default_rng(616)
    C = 30_000
    contig = _rand(rng, C)
    jobs = []
    for R, a, L in ((400, 120, 150), (1200, 0, 300), (2500, 1900, 600), (900, 400, 500), (3000, 2990, 10)):
        o = int(rng.integers(1000, C - R - 1000))
        jobs.append((o + a, L, o, R))
    for R, L in ((800, 200), (1500, 400)):
        o = int(rng.integers(1000, C - R - 1000))
        jobs.append((o - L // 2, L, o, R))
        jobs.append((o + R - L // 2, L, o, R))
    b = _batch(contig, jobs)
    ok, _, rows = ctx.long_needle(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"])
    for i in range(len(jobs)):
        eok, e0, e1 = po.long_needle(ref, _seq(b, i, "q"), _seq(b, i, "t"))
        assert bool(ok[i]) == eok, i
        if eok:
            assert rows[i] == (e0, e1), i


@pytest.mark.gpu
def test_msa_shared_arena_bytes(ctx, ref):
    """MSA clusters whose reads are overlapping windows of one region of the arena, some of them the very same bytes."""
    rng = np.random.default_rng(717)
    contig = _rand(rng, 20_000)
    read_off, read_len, coff = [], [], [0]
    for _ in range(8):
        o, L = int(rng.integers(0, 19_000)), int(rng.integers(90, 240))
        for r in range(int(rng.integers(3, 12))):
            s = o + int(rng.integers(0, 60)) if r % 3 else o
            read_off.append(s); read_len.append(min(L + int(rng.integers(-20, 20)), 20_000 - s))
        coff.append(len(read_off))
    ro, rl = np.array(read_off, np.uint32), np.array(read_len, np.uint32)
    cons, nrows, status = ctx.msa(contig, ro, rl, np.array(coff, np.uint32))
    for i in range(len(coff) - 1):
        reads = [contig[int(ro[r]):int(ro[r]) + int(rl[r])].tobytes() for r in range(coff[i], coff[i + 1])]
        erows, ecs, _ = po.msa(ref, reads, 2)
        assert cons[i] == ecs and nrows[i] == erows, i


# ---------------------------------------------------------------------------------------------------------------------------------------
# 2-4. target slices of 4 kb to the 16384-column limit, deep Hirschberg recursion

def _slice_batch(mode, eq):
    """Pairs whose aligned target slice is each of SLICES (5-12 % divergence: band classes G = 16 and 32), unrelated pairs (no band
    certifies them: wavefront classes 9-11), and for NW queries of <= 128 bases against 4-16 kb targets (unsplit class-10/11 leaves)."""
    rng = np.random.default_rng(8100 + 10 * mode + len(eq))
    seqs = []
    for i, L in enumerate(SLICES):
        rate = 0.05 + 0.07 * i / (len(SLICES) - 1)
        pad = (0, 0) if mode == 0 else (0, 1500) if mode == 1 else (1500, 1500)
        base = _rand(rng, pad[0] + L + pad[1])
        q = _noisy(rng, base[pad[0]:pad[0] + L], rate)
        t = base
        if eq:   # IUPAC bytes everywhere but at the slice's ends, which stay exact like the query's flanks
            t = _sprinkle(rng, base)
            for e in (pad[0], pad[0] + L - 32):
                t[e:e + 32] = base[e:e + 32]
        seqs += [q, t]
    if mode == 0:
        for L in (4097, 8192, 16384):
            seqs += [_rand(rng, L - int(rng.integers(0, 400))), _rand(rng, L)]
        for L in (4097, 8192, 8193, 12000, 16383, 16384):
            seqs += [_rand(rng, int(rng.integers(40, 129))), _rand(rng, L)]
    else:
        for L in (5000, 9500):
            seqs += [_rand(rng, L), _rand(rng, L + 2000)]
    if eq:
        for j in range(len(seqs) // 2):
            if j >= len(SLICES):
                seqs[2 * j + 1] = _sprinkle(rng, seqs[2 * j + 1])
    return _packed(seqs)


@pytest.mark.gpu
@EQS
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_path_slice_classes(ctx, ref, mode, eq):
    """Aligned target slices on and between the segment class boundaries 4096 / 8192 / 16384, in every mode, with and without the pairs."""
    b = _slice_batch(mode, eq)
    res = _check_paths(ctx, ref, b, mode, eq)
    slices = {re - rs + 1 for _, re, rs in res}
    assert set(SLICES) <= slices, sorted(slices)
    if mode == 0:   # an unsplit NW leaf of 20 ceil(m/64) n + 8 n < 2^20 bytes over more than 8192 columns
        assert any(ln <= 128 and tl > 8192 and 20 * ((ln + 63) // 64) * tl + 8 * tl < 1 << 20 for ln, tl in zip(b["q_len"], b["t_len"]))


@pytest.mark.gpu
def test_path_msaedlib_long_consensus(ctx, ref):
    """msaEdlib's call at long-read sizes: a read against a gapped IUPAC consensus of 8-16 kb, NW with the 20 pairs."""
    rng = np.random.default_rng(909)
    seqs = []
    for L in (8000, 11000, 13500, 15600):
        base = _rand(rng, L)
        read = synth.mutate_fast(rng, base, sub=0.03, ins=0.02, dele=0.02)
        cons = _sprinkle(rng, base, 0.03)
        gaps = np.sort(rng.choice(L, size=L // 25, replace=False))
        cons = np.insert(cons, gaps, np.uint8(ord("-")))
        seqs += [read, cons[:SLICE_LIMIT]]
    _check_paths(ctx, ref, _packed(seqs), 0, IUPAC_EQ)


def _depth_lb(m, n):
    """Fewest recursion levels (leaves included) Hirschberg's split can give an m x n problem, whatever rows it splits at: the 1 MiB test
    (src/edlib.cpp:1189-1191) grows with m and n, and one child keeps at least half the rows and half the columns (rounded down)."""
    lv = 1
    while 20 * ((m + 63) // 64) * n + 8 * n >= 1 << 20:
        m, n, lv = (m + 1) // 2, n // 2, lv + 1
    return lv


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])
def test_path_deep_hirschberg(ctx, ref, mode):
    """Problems of 14.6-16.4 kb on both sides: at least five levels of recursion, with ACG repeats so that ties decide at every level."""
    rng = np.random.default_rng(1212 + mode)
    acg = lambda n: np.resize(np.frombuffer(b"ACG", np.uint8), n)
    seqs = []
    if mode == 0:
        for m, n, kind in ((16000, 16384, "rep"), (15100, 14700, "rep"), (16200, 16200, "sim"), (14800, 15900, "sim")):
            if kind == "rep":
                seqs += [acg(m), acg(n)]
            else:
                t = _rand(rng, n)
                seqs += [synth.mutate_fast(rng, t, sub=0.05, ins=0.02, dele=0.02)[:m], t]
    else:
        t = _rand(rng, 22_000)
        seqs += [_noisy(rng, t[3000:18_500], 0.08), t, acg(15_000), acg(21_000)]
    b = _packed(seqs)
    res = _check_paths(ctx, ref, b, mode, b"")
    for i, (_, re, rs) in enumerate(res):
        assert _depth_lb(int(b["q_len"][i]), re - rs + 1) >= 5, (i, int(b["q_len"][i]), re - rs + 1)


@pytest.mark.gpu
@EQS
def test_path_slice_limit_nw(ctx, ref, eq):
    """NW: a 16384-column target is traced; a 16385-column one gets status 2 alone (no ops, the reference's distance and locations)."""
    rng = np.random.default_rng(1313 + len(eq))
    seqs, status = [], []
    for n, st, kind in ((16384, 0, "sim"), (16385, 2, "sim"), (700, 0, "sim"), (16385, 2, "short"), (2500, 0, "sim"), (16384, 0, "short")):
        t = _rand(rng, n)
        q = synth.mutate_fast(rng, t, sub=0.02, ins=0.01, dele=0.01) if kind == "sim" else _rand(rng, 120)
        seqs += [q, _sprinkle(rng, t) if eq else t]
        status.append(st)
    _check_paths(ctx, ref, _packed(seqs), 0, eq, status)


@pytest.mark.gpu
@EQS
def test_path_slice_limit_hw(ctx, ref, eq):
    """HW: queries inside a 40 kb target (some of them its own bytes): a 16384-column slice is traced, a 16385-column one gets status 2,
    and the small jobs of the batch are unaffected."""
    rng = np.random.default_rng(1414 + len(eq))
    T = 40_000
    t = _rand(rng, T)
    if eq:
        t = _sprinkle(rng, t)
    reads, jobs, status = [], [], []
    off = T
    for a, L, inside in ((5000, SLICE_LIMIT, True), (21_000, SLICE_LIMIT + 1, True), (300, SLICE_LIMIT, False), (12_000, SLICE_LIMIT + 1, False),
                         (30_000, 900, False), (100, 64, True)):
        if inside:
            jobs.append((a, L, 0, T))
        else:
            r = _noisy(rng, t[a:a + L], 0.02)
            jobs.append((off, len(r), 0, T))
            reads.append(r)
            off += len(r)
        status.append(2 if L > SLICE_LIMIT else 0)
    res = _check_paths(ctx, ref, _batch(np.concatenate([t] + reads), jobs), 2, eq, status)
    assert [re - rs + 1 for _, re, rs in res][:4] == [SLICE_LIMIT, SLICE_LIMIT + 1, SLICE_LIMIT, SLICE_LIMIT + 1]


@pytest.mark.gpu
def test_path_long_slices_without_band_passes():
    """The slice, Hirschberg and limit batches above once more with DGPU_EP_NO_BAND=1 (read once per process), which sends every segment
    through the wavefront kernels, classes 1-11. They run in a child pytest that has exited when this test returns."""
    if os.environ.get("DGPU_EP_NO_BAND"):
        pytest.skip("this is the child run")
    env = dict(os.environ, DGPU_EP_NO_BAND="1")
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", "-k", "slice_classes or hirschberg or slice_limit or msaedlib",
           os.path.abspath(__file__)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout, r.stdout[-2000:]


# ---------------------------------------------------------------------------------------------------------------------------------------
# 6. multi-stripe edit distances (|q| > 2048: ed_long_kernel hands each 2048-row stripe's last row to the next through global scratch)

QLENS = [2049, 4095, 4097, 6144, 10000, 20000]


def _stripe_batch():
    """Per query length: a query drawn from a longer target (up to 40 kb), an unrelated pair, and a target shorter than the query."""
    rng = np.random.default_rng(2020)
    seqs = []
    for L in QLENS:
        n = min(40_000, L + int(rng.integers(100, 20_000)))
        t = _rand(rng, n)
        a = int(rng.integers(0, n - L + 1))
        seqs += [synth.mutate_fast(rng, t[a:a + L], sub=0.04, ins=0.02, dele=0.02), t]
        seqs += [_rand(rng, L), _rand(rng, int(rng.integers(L, 40_001)))]
        seqs += [_rand(rng, L), _rand(rng, int(rng.integers(L // 2, L)))]
    seqs += [_rand(rng, 20_000), _rand(rng, 40_000)]
    return _packed(seqs)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_distance_multi_stripe(ctx, oracle, mode):
    """Queries of 2049-20000 bases against targets of up to 40 kb, with end locations and k unbounded, below, at and above the distance;
    then the same with dgpu_set_async_bound(40000), where the stripe scratch is sized from the bound instead of the batch."""
    b = _stripe_batch()
    n = len(b["q_off"])
    assert b["t_len"].max() <= 40_000 and b["q_len"].max() <= 40_000
    threads = os.cpu_count() or 1
    args = (b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"])
    od, oe = po.edit_distance_batch(oracle, *args, None, mode, threads=threads, want_end=True)
    # k = -1, d - 1, d, d + 1 for every job, as one batch of 4 n jobs
    k = np.concatenate([np.full(n, -1), np.maximum(od - 1, 0), od, od + 1]).astype(np.int32)
    tiled = (b["seqs"],) + tuple(np.tile(b[c], 4) for c in ("q_off", "q_len", "t_off", "t_len"))
    kd, ke = po.edit_distance_batch(oracle, *tiled, k, mode, threads=threads, want_end=True)
    assert np.array_equal(kd[:n], od) and (kd[n:2 * n] == -1).any()
    gd, ge = ctx.edit_distance(*args, None, mode, want_end=True)
    assert np.array_equal(gd, od) and np.array_equal(ge, oe)
    lib = delly_b200.lib()
    for bound in (0, 40_000):
        ctx.check(lib.dgpu_set_async_bound(ctx.h, bound), "dgpu_set_async_bound")
        try:
            gd, ge = ctx.edit_distance(*tiled, k, mode, want_end=True)
        finally:
            ctx.check(lib.dgpu_set_async_bound(ctx.h, 0), "dgpu_set_async_bound")
        assert np.array_equal(gd, kd), (bound, np.nonzero(gd != kd)[0][:8])
        assert np.array_equal(ge, ke), (bound, np.nonzero(ge != ke)[0][:8])
