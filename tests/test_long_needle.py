"""longNeedle (src/needle.h:45-222): oracle vs compiled reference (CPU), CUDA vs oracle / golden (GPU)."""
import os

import numpy as np
import pytest

from delly_b200 import synth
from oracle import pyoracle as po

GOLD = os.path.join(os.path.dirname(__file__), "golden", "long_needle.npz")


def _jobs(b):
    for i in range(len(b["c_off"])):
        c = b["seqs"][b["c_off"][i]: b["c_off"][i] + b["c_len"][i]].tobytes()
        r = b["seqs"][b["r_off"][i]: b["r_off"][i] + b["r_len"][i]].tobytes()
        yield c, r


def _edge_batch(seed=3):
    """Degenerate and adversarial inputs: empty, single base, homopolymers/repeats (many ties), N / IUPAC / lower case."""
    rng = np.random.default_rng(seed)
    A = lambda n: synth._ACGT[rng.integers(0, 4, size=n)]  # noqa: E731
    seqs = [b"", b"ACGT", b"ACGT", b"", b"A", b"A", b"A", b"C", b"ACGTACGTAC", b"ACGTACGTAC",
            b"A" * 40, b"A" * 90, b"AC" * 30, b"AC" * 70, b"ACG" * 20, b"ACG" * 9 + b"TTTTTTTTTTTTTTTTTTTT" + b"ACG" * 20]
    for _ in range(40):
        n = int(rng.integers(1, 140)); m = int(rng.integers(1, 60))
        r = A(n)
        if rng.random() < 0.5 and n > 30:
            a = int(rng.integers(0, n // 2)); b = int(rng.integers(n // 2, n))
            c = np.concatenate([r[max(0, a - m):a], r[b:b + m]])
        else:
            c = A(m)
        if rng.random() < 0.4:
            c = c.copy(); r = r.copy()
            for arr in (c, r):
                if len(arr):
                    for p in rng.integers(0, len(arr), size=max(1, len(arr) // 8)):
                        arr[p] = rng.choice(np.frombuffer(b"NNRYacgtnM", np.uint8))
        seqs += [c, r]
    arena, off, ln = synth.pack(seqs)
    return dict(seqs=arena, c_off=off[0::2].copy(), c_len=ln[0::2].copy(), r_off=off[1::2].copy(), r_len=ln[1::2].copy())


def test_oracle_matches_reference(ref):
    O = po.oracle()
    nt = nf = 0
    for b in (synth.k3_consref_batch(120, seed=5, cons_range=(40, 120), ref_cap=500), _edge_batch()):
        for c, r in _jobs(b):
            if len(c) == 0 or len(r) == 0:
                continue  # the reference itself is only defined for non-empty inputs here
            a = po.long_needle(O, c, r)
            e = po.long_needle(ref, c, r)
            assert a == e, (len(c), len(r))
            nt += a[0]; nf += (not a[0])
    assert nt > 60 and nf > 10


def test_golden_long_needle(oracle):
    g = np.load(GOLD)
    b = {k: g[k] for k in ("seqs", "c_off", "c_len", "r_off", "r_len")}
    for i, (c, r) in enumerate(_jobs(b)):
        ok, r0, r1 = po.long_needle(oracle, c, r)
        assert int(ok) == g["ok"][i]
        if ok:
            o, L = int(g["aln_off"][i]), int(g["aln_len"][i])
            assert r0 == g["aln"][o:o + L].tobytes() and r1 == g["aln"][o + L:o + 2 * L].tobytes()


def _check_against_oracle(ctx, b, threads=8):
    ok, alen, rows = ctx.long_needle(b["seqs"], b["c_off"], b["c_len"], b["r_off"], b["r_len"])
    O = po.oracle()
    nt = 0
    for i, (c, r) in enumerate(_jobs(b)):
        eok, e0, e1 = po.long_needle(O, c, r)
        assert bool(ok[i]) == eok, (i, len(c), len(r))
        if eok:
            assert rows[i][0] == e0, (i, len(c), len(r))
            assert rows[i][1] == e1, (i, len(c), len(r))
            nt += 1
    return nt


@pytest.mark.gpu
def test_cuda_edges(ctx):
    _check_against_oracle(ctx, _edge_batch())


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [((40, 120), 500, 150), ((150, 300), None, 60), ((150, 300), 1000, 40), ((400, 700), 3000, 10), ((900, 1200), 5000, 4),
                                   ((1500, 2100), None, 3), ((2600, 3400), None, 3)])   # long-read shapes: 4-warp / 8-warp CTAs, C = 32 and C = 64
def test_cuda_matches_oracle(ctx, shape):
    cr, cap, n = shape
    b = synth.k3_consref_batch(n, seed=11 + cr[0], cons_range=cr, ref_cap=cap)
    nt = _check_against_oracle(ctx, b)
    assert nt >= n // 2


@pytest.mark.gpu
def test_cuda_golden(ctx):
    g = np.load(GOLD)
    ok, alen, rows = ctx.long_needle(g["seqs"], g["c_off"], g["c_len"], g["r_off"], g["r_len"])
    assert np.array_equal(ok, g["ok"])
    for i in range(len(ok)):
        if ok[i]:
            o, L = int(g["aln_off"][i]), int(g["aln_len"][i])
            assert rows[i][0] == g["aln"][o:o + L].tobytes() and rows[i][1] == g["aln"][o + L:o + 2 * L].tobytes()


@pytest.mark.gpu
def test_cuda_widest_windows(ctx):
    """The widest reference windows the device path takes (n + 7 <= 16384): the 8-warp CTAs with 56 and 64 columns per lane,
    whose row state lives in shared memory. Deletion-like split of the consensus, substitution noise."""
    rng = np.random.default_rng(99)
    seqs = []
    for n, m in ((14400, 2600), (15011, 3300), (16377, 2900)):
        ref = synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]
        a = int(rng.integers(100, n // 3)); b = int(rng.integers(2 * n // 3, n - m))
        cons = synth.sub_noise(rng, np.concatenate([ref[a:a + m // 2], ref[b:b + (m - m // 2)]]), 0.03)
        seqs += [cons, ref]
    arena, off, ln = synth.pack(seqs)
    b = dict(seqs=arena, c_off=off[0::2].copy(), c_len=ln[0::2].copy(), r_off=off[1::2].copy(), r_len=ln[1::2].copy())
    assert _check_against_oracle(ctx, b) == 3


@pytest.mark.gpu
def test_cuda_oversize_job_fails_alone(ctx):
    """A window beyond the kernel's shapes (|ref| > 16377) inside a normal batch: that ONE job comes back not aligned (ok = 0), the call
    succeeds and every other job equals the reference (VERDICT r1 item 8: no batch-aborting limits)."""
    import delly_b200
    rng = np.random.default_rng(41)
    b = synth.k3_consref_batch(24, seed=9, cons_range=(80, 160), ref_cap=700)
    jobs = list(_jobs(b))
    big_ref = synth._ACGT[rng.integers(0, 4, size=17000)].tobytes()
    big_cons = big_ref[3000:3100] + big_ref[9000:9100]
    jobs.insert(7, (big_cons, big_ref))
    seqs = [x for cr in jobs for x in cr]
    arena, off, ln = synth.pack(seqs)
    before = ctx._lib.dgpu_unsupported_count
    before.restype = delly_b200.C.c_uint64
    n0 = before(ctx.h)
    ok, alen, rows = ctx.long_needle(arena, off[0::2].copy(), ln[0::2].copy(), off[1::2].copy(), ln[1::2].copy())
    assert before(ctx.h) == n0 + 1
    assert ok[7] == 0 and alen[7] == 0
    O = po.oracle()
    for i, (c, r) in enumerate(jobs):
        if i == 7:
            continue
        eok, e0, e1 = po.long_needle(O, c, r)
        assert bool(ok[i]) == eok and (not eok or (rows[i][0] == e0 and rows[i][1] == e1)), i


@pytest.mark.gpu
def test_cuda_non_acgtn_jobs_take_the_scalar_engine(ctx):
    """jobs with IUPAC / lower-case bytes are routed to the byte-comparing engine, ACGTN jobs to the packed one: one mixed batch, all equal the oracle"""
    O = po.oracle()
    b1 = synth.k3_consref_batch(40, seed=12, cons_range=(60, 200), ref_cap=900)
    b2 = _edge_batch(seed=5)
    jobs = [j for j in list(_jobs(b1)) + list(_jobs(b2)) if len(j[0]) and len(j[1])]
    # one job on each side of every class bound on n + 7, over ACGTN (packed engine) and with one lower-case byte (scalar engine)
    rng = np.random.default_rng(77)
    bounds = [b for k in range(1, 9) for b in (256 * k, 256 * k + 1)] + [b for k in range(4096, 16384, 2048) for b in (k, k + 1)] + [16384]
    for n in (b - 7 for b in bounds):
        ref = synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]
        a = int(rng.integers(0, n // 3)); b = int(rng.integers(2 * n // 3, n - 60))
        cons = synth.sub_noise(rng, np.concatenate([ref[a:a + 60], ref[b:b + 60]]), 0.03)
        low = ref.copy()
        low[n // 2] += 32
        jobs += [(cons.tobytes(), ref.tobytes()), (cons.tobytes(), low.tobytes())]
    arena, off, ln = synth.pack([x for cr in jobs for x in cr])
    ok, alen, rows = ctx.long_needle(arena, off[0::2].copy(), ln[0::2].copy(), off[1::2].copy(), ln[1::2].copy())
    for i, (c, r) in enumerate(jobs):
        eok, e0, e1 = po.long_needle(O, c, r)
        assert bool(ok[i]) == eok and (not eok or (rows[i][0] == e0 and rows[i][1] == e1)), (i, len(c), len(r))
