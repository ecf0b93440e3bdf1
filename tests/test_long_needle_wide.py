"""longNeedle (src/needle.h:45-222) on reference windows beyond the wavefront kernels' shapes (|ref| > 16377 or |cons| + |ref| > 32000):
the wide-window engine of dgpu_long_needle_ex against the oracle (GPU), its refusals and argument checks, and the long-read call chain with
deletions of 12-30 kb, whose consensus windows cross both limits, against the reference (GPU, and on the CPU through the test stand-in)."""
import ctypes as C
import os

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po
from test_bcf_parity import DELLY_REF, EX, ROOT, _inflate, _run
from test_host_genotype import LR_CFG
from test_host_split import _p
from test_msa_large import _build_standin

_wide_job = synth.wide_consref_job


def _batch(jobs):
    arena, off, ln = synth.pack([x for cr in jobs for x in cr])
    return arena, off[0::2].copy(), ln[0::2].copy(), off[1::2].copy(), ln[1::2].copy()


def _check(ctx, jobs, max_ref=delly_b200.LN_MAX_REF):
    """CUDA (dgpu_long_needle_ex) against the oracle on every job; returns the number of true results."""
    arena, co, cl, ro, rl = _batch(jobs)
    ok, alen, rows, info = ctx.long_needle(arena, co, cl, ro, rl, want_info=True, max_ref=max_ref)
    O = po.oracle()
    nt = 0
    for i, (c, r) in enumerate(jobs):
        eok, e0, e1 = po.long_needle(O, bytes(c), bytes(r))
        assert info[i][2] != -1 or len(c) == 0, (i, len(c), len(r))   # not refused
        assert bool(ok[i]) == eok, (i, len(c), len(r))
        if eok:
            assert rows[i][0] == e0 and rows[i][1] == e1, (i, len(c), len(r), info[i].tolist())
            nt += 1
    return nt


def _unsupported(ctx):
    f = ctx._lib.dgpu_unsupported_count
    f.restype = C.c_uint64
    return int(f(ctx.h))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,m,n", [("del", 1000, 16378), ("del", 1500, 24000), ("del", 3000, 40000), ("dup", 4500, 18000), ("inv", 5000, 20000),
                                      ("dup", 6000, 16900), ("del", 2500, 30000), ("inv", 1200, 33000)])
def test_cuda_wide_matches_oracle(ctx, kind, m, n):
    """DEL-, DUP- and INV-shaped windows of 16378 to 40000 columns, consensus of 1-6 kb (the last three: |cons| + |ref| > 32000)"""
    rng = np.random.default_rng(m + n)
    jobs = [_wide_job(rng, kind, m, n), _wide_job(rng, kind, m, n, noise=0.08)]
    jobs.append((synth._ACGT[rng.integers(0, 4, size=m, dtype=np.uint8)], jobs[0][1]))   # unrelated consensus: no split found
    assert _check(ctx, jobs) >= 2


@pytest.mark.gpu
def test_cuda_wide_non_acgt_bytes(ctx):
    """N, IUPAC and lower-case bytes in either sequence (the engine compares bytes; the reverse part follows reverseComplement's rule, which
    leaves other bytes in place, so that dense IUPAC codes make the two passes disagree and longNeedle return false)"""
    rng = np.random.default_rng(5)
    jobs = []
    for k, (m, n) in enumerate(((1800, 17000), (2200, 21000), (1500, 26000))):
        c0, r0 = _wide_job(rng, ("del", "dup", "inv")[k], m, n)
        for alphabet, frac in ((b"N", 40), (b"NNRYacgtnMKWS", 1000), (b"NNRYacgtnMKWS", 400), (b"NNRYacgtnMKWS", 40)):
            c, r = c0.copy(), r0.copy()
            for arr, f in ((c, frac), (r, 10 * frac)):
                pos = rng.integers(0, len(arr), size=len(arr) // f)
                arr[pos] = rng.choice(np.frombuffer(alphabet, np.uint8), size=len(pos))
            jobs.append((c, r))
    assert _check(ctx, jobs) >= 4


def _lnw_grids(n):
    """lnw_kernel's column grids for a window of n columns (lnw_geom): the reverse grid starts at column o = n mod 8 in [-6, 1], the forward
    grid at 1; thread t of either pass owns the J (odd) chunks of 8 columns that start at origin + 8*J*t."""
    o = 1 - ((1 - n) & 7)
    nqR = (n - o) // 8 + 1
    J = ((nqR + 511) // 512) | 1
    return o, J


@pytest.mark.gpu
def test_cuda_wide_breakpoints_on_thread_boundaries(ctx):
    """Deletion-shaped jobs whose left breakpoint (the best join's refLeft) sits on the first column of a forward-pass thread segment or
    just before it, and whose right breakpoint (refRight, counted from the end in the reverse pass) sits on the first column of a
    reverse-pass thread segment or just before it; windows of every residue mod 8 (reverse grid origins 1, 0, -1 .. -6) and at column 16384,
    where the wavefront kernels end"""
    rng = np.random.default_rng(17)
    jobs = []
    h = 600
    for n in [20000 + k for k in range(8)] + [40001, 40004, 24007]:
        o, J = _lnw_grids(n)
        seg = 8 * J
        for t, d in ((20, 0), (33, -1), (47, 0), (61, 1)):
            a = 1 + seg * t + d                    # forward columns 1 .. a on the left of the join
            x = o + seg * (t + 20) + d             # reverse column of the right breakpoint: refRight = n - b
            b = n - x
            g = synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]
            jobs.append((synth.sub_noise(rng, np.concatenate([g[a - h:a], g[b:b + h]]), 0.01), g))
    g = synth._ACGT[rng.integers(0, 4, size=18000, dtype=np.uint8)]
    jobs.append((np.concatenate([g[16384 - h:16384], g[17000:17000 + h]]), g))
    assert _check(ctx, jobs) >= len(jobs) - 2


@pytest.mark.gpu
def test_cuda_wide_device_form(ctx):
    """dgpu_long_needle_ex_dev (Context.long_needle_dev with max_ref) on device tensors: wide and ordinary jobs equal the oracle"""
    import torch
    rng = np.random.default_rng(29)
    small = synth.k3_consref_batch(8, seed=7, cons_range=(100, 200), ref_cap=800)
    jobs = [(small["seqs"][small["c_off"][i]:small["c_off"][i] + small["c_len"][i]], small["seqs"][small["r_off"][i]:small["r_off"][i] + small["r_len"][i]])
            for i in range(8)]
    jobs[2:2] = [_wide_job(rng, "del", 1500, 21003)]
    jobs[6:6] = [_wide_job(rng, "inv", 2500, 30001)]
    arena, co, cl, ro, rl = _batch(jobs)
    cap = cl.astype(np.uint64) + rl.astype(np.uint64)
    aoff = np.concatenate([[0], np.cumsum(2 * cap)[:-1]]).astype(np.uint64)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()   # noqa: E731
    aln = torch.zeros(int(2 * cap.sum()), dtype=torch.uint8, device="cuda")
    alen = torch.zeros(len(jobs), dtype=torch.int32, device="cuda")
    ok = torch.zeros(len(jobs), dtype=torch.uint8, device="cuda")
    n0 = _unsupported(ctx)
    ctx.long_needle_dev(dev(arena), dev(co.view(np.int32)), dev(cl.view(np.int32)), dev(ro.view(np.int32)), dev(rl.view(np.int32)), aln,
                        dev(aoff.view(np.int64)), alen, ok, max_ref=30001)
    ctx.sync()
    assert _unsupported(ctx) == n0
    aln, alen, ok = aln.cpu().numpy(), alen.cpu().numpy(), ok.cpu().numpy()
    O = po.oracle()
    for i, (c, r) in enumerate(jobs):
        eok, e0, e1 = po.long_needle(O, bytes(c), bytes(r))
        assert bool(ok[i]) == eok, i
        if eok:
            o, L, k = int(aoff[i]), int(alen[i]), int(cap[i])
            assert aln[o:o + L].tobytes() == e0 and aln[o + k:o + k + L].tobytes() == e1, i
    assert ok[2] and ok[6]


@pytest.mark.gpu
def test_cuda_wide_equal_joins_far_apart(ctx):
    """Two copies of the consensus's right half in the window, thousands of columns apart: joins of equal score in different thread
    segments and rows, where the first maximum in row-major order must win (needle.h:104-115) and refRight is the last equal right bound"""
    rng = np.random.default_rng(23)
    jobs = []
    for n, gap in ((20000, 6000), (36000, 15000), (30000, 8 * 5 * 97)):
        g = synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]
        rep = g[n - 900:n - 300].copy()
        g[n - 900 - gap:n - 300 - gap] = rep       # the same 600 bases twice
        cons = np.concatenate([g[400:1000], rep])
        jobs.append((cons, g))
        jobs.append((np.concatenate([rep, g[n - 300:]]), g))
    assert _check(ctx, jobs) >= len(jobs) // 2


@pytest.mark.gpu
def test_cuda_wide_mixed_with_ordinary_jobs(ctx):
    """Wide jobs inside a batch of ordinary K3 (short-read) and K5 (long-read) jobs: every result equals the oracle"""
    rng = np.random.default_rng(31)
    b3 = synth.k3_consref_batch(60, seed=3, cons_range=(80, 250), ref_cap=900)
    b5 = synth.k3_consref_batch(6, seed=5, cons_range=(1500, 3000), ref_cap=None)
    jobs = []
    for b in (b3, b5):
        for i in range(len(b["c_off"])):
            jobs.append((b["seqs"][b["c_off"][i]:b["c_off"][i] + b["c_len"][i]], b["seqs"][b["r_off"][i]:b["r_off"][i] + b["r_len"][i]]))
    for k, (kind, m, n) in enumerate((("del", 2000, 22000), ("inv", 3000, 17000), ("del", 1500, 31000))):
        jobs.insert(7 + 20 * k, _wide_job(rng, kind, m, n))
    n0 = _unsupported(ctx)
    _check(ctx, jobs)
    assert _unsupported(ctx) == n0


@pytest.mark.gpu
def test_cuda_wide_refusals(ctx):
    """Jobs beyond max_ref, and a consensus beyond 16383 bases, are refused alone (ok = 0, info[2] = -1, counted); the old entry point still
    refuses every wide job; max_ref outside 1 .. DGPU_LN_MAX_REF is an argument error"""
    rng = np.random.default_rng(41)
    small = synth.k3_consref_batch(12, seed=9, cons_range=(80, 160), ref_cap=700)
    jobs = [(small["seqs"][small["c_off"][i]:small["c_off"][i] + small["c_len"][i]], small["seqs"][small["r_off"][i]:small["r_off"][i] + small["r_len"][i]])
            for i in range(12)]
    w1 = _wide_job(rng, "del", 1500, 20000)
    w2 = _wide_job(rng, "del", 1500, 26000)
    big_cons = (synth._ACGT[rng.integers(0, 4, size=16400, dtype=np.uint8)], synth._ACGT[rng.integers(0, 4, size=17000, dtype=np.uint8)])
    jobs[3:3] = [w1]
    jobs[8:8] = [w2]
    jobs.append(big_cons)
    arena, co, cl, ro, rl = _batch(jobs)
    O = po.oracle()
    n0 = _unsupported(ctx)
    ok, alen, rows, info = ctx.long_needle(arena, co, cl, ro, rl, want_info=True, max_ref=22000)   # w2 (26000) beyond max_ref
    assert _unsupported(ctx) == n0 + 2
    for i, (c, r) in enumerate(jobs):
        if i in (8, len(jobs) - 1):
            assert ok[i] == 0 and alen[i] == 0 and info[i][2] == -1, i
            continue
        eok, e0, e1 = po.long_needle(O, bytes(c), bytes(r))
        assert bool(ok[i]) == eok and (not eok or (rows[i][0] == e0 and rows[i][1] == e1)), i
    # the old entry point: every job beyond its shapes is refused, the others are computed
    n0 = _unsupported(ctx)
    ok2, alen2, rows2 = ctx.long_needle(arena, co, cl, ro, rl)
    assert _unsupported(ctx) == n0 + 3
    for i in (3, 8, len(jobs) - 1):
        assert ok2[i] == 0 and alen2[i] == 0
    assert all(rows2[i] == rows[i] for i in range(len(jobs)) if i not in (3, 8, len(jobs) - 1))
    for bad in (0, delly_b200.LN_MAX_REF + 1):
        with pytest.raises(delly_b200.DgpuError, match="max_ref"):
            ctx.long_needle(arena, co, cl, ro, rl, max_ref=bad)


# ---- the long-read call chain with large deletions -------------------------------------------------------------------------------

def _simulate_lr_large_dels(seed, sizes=(12500, 15500, 18000, 22000, 26000, 30000), cov=14):
    """A diploid sample (as test_host_genotype._simulate_lr_sample) with large heterozygous / homozygous deletions on contig 0, 2-5 kb reads
    with 5 % substitutions; a read over a deletion carries it as a D operation of its CIGAR."""
    rng = np.random.default_rng(seed)
    L0 = 60000 + 48000 * len(sizes)
    ref0 = synth._ACGT[rng.integers(0, 4, size=L0, dtype=np.uint8)]; ref1 = synth._ACGT[rng.integers(0, 4, size=20000, dtype=np.uint8)]
    starts = [20000 + 48000 * i + int(rng.integers(0, 2000)) for i in range(len(sizes))]
    zyg = rng.choice([1, 2], size=len(sizes), p=[0.5, 0.5])
    recs, cigs, reads = [], [], []
    total = int(L0 * cov / 3500)
    for rid in range(total):
        tid = 0 if rng.random() < 0.92 else 1
        L = int(rng.integers(2000, 5001))
        hap = int(rng.integers(0, 2))
        G = ref0 if tid == 0 else ref1
        p = int(rng.integers(0, len(G) - L - 2000))
        ops, seq, rp, left = [], [], p, L
        ev = [(s, z) for s, z, g in zip(starts, sizes, zyg) if tid == 0 and (g == 2 or hap == 1) and s > p + 300]
        for s, z in ev:
            if s - rp >= left - 300:
                break
            ops.append((0, s - rp)); seq.append(G[rp:s]); left -= s - rp; rp = s + z
            ops.append((2, z))
        if rp + left > len(G):
            continue
        ops.append((0, left)); seq.append(G[rp:rp + left])
        s = synth.sub_noise(rng, np.concatenate(seq), 0.05)
        flag = int(rng.choice([0, 16]))
        recs.append([tid, p, flag, 60, len(s), len(cigs), len(ops), sum(len(r) for r in reads), tid, 0, 0, rid])
        cigs.extend((ln << 4) | op for op, ln in ops)
        reads.append(s)
    r = np.array(recs, np.int64)
    order = np.lexsort((np.arange(len(r)), r[:, 1], r[:, 0]))
    return dict(contig=np.concatenate([ref0, ref1]), coff=np.array([0, L0], np.uint32), clen=np.array([L0, len(ref1)], np.uint32),
                rec=np.ascontiguousarray(r[order].astype(np.int32)), cig=np.array(cigs, np.uint32), reads=np.concatenate(reads).astype(np.uint8),
                truth=list(zip(starts, sizes)))


@pytest.fixture(params=[pytest.param("gpu", marks=pytest.mark.gpu), "edlib-standin"])
def hostdev_wide(request, ref):
    """(host library, context handle): the real libraries on an H100, or the CPU stand-in with dgpu_long_needle_ex forwarded to the
    reference's longNeedle"""
    if request.param == "gpu":
        return delly_b200.hostlib(), request.getfixturevalue("ctx")
    lib = C.CDLL(_build_standin("libhost_standin_long_needle_ex.so", ["host_standin.cpp", "long_needle_ex_standin.cpp"], shared=True))
    lib.standin_ctx.restype = C.c_void_p
    return lib, None


def test_delly_lr_call_large_deletions_match_reference(hostdev_wide, ref5):
    """`delly lr -i 40000` on deletions of 12-30 kb: consensus windows beyond 16377 columns and beyond |cons| + |ref| = 32000. Every record
    field equals the reference's; on the GPU no consensus alignment is refused"""
    H, ctx = hostdev_wide
    ctxh = ctx.h if ctx is not None else C.c_void_p(H.standin_ctx())
    d = _simulate_lr_large_dels(2024)
    nrec = len(d["rec"])
    cfg = LR_CFG.copy()
    cfg[8] = 40000   # indelsize
    ref5.ref_hash_lr_name5.restype = C.c_uint64
    seeds = np.array([ref5.ref_hash_lr_name5(f"q{int(r[11])}".encode()) for r in d["rec"]], np.uint64)
    n0 = _unsupported(ctx) if ctx is not None else 0
    outs = []
    for which in ("ref", "ours"):
        sv = np.zeros((512, 20), np.int32); fmt = np.zeros((512, 14), np.int32); gl = np.zeros((512, 3), np.float32)
        co = np.zeros((512, 16384), np.uint8); cl = np.zeros(512, np.int32)
        tail = (_p(d["cig"]), _p(d["reads"]), _p(cfg), C.c_float(0.9), C.c_float(0.5), _p(sv), 512, _p(fmt), _p(gl), _p(co), 16384, _p(cl))
        if which == "ref":
            n = ref5.ref_delly_lr_call(_p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 2, _p(d["rec"]), nrec, *tail)
        else:
            n = H.dh_delly_lr_call(ctxh, _p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 2, _p(d["rec"]), _p(seeds), nrec, *tail)
        assert n > 0, n
        outs.append((n, sv[:n].copy(), fmt[:n].copy(), gl[:n].copy(), [co[i, :cl[i]].tobytes() for i in range(n)]))
    e, g = outs
    assert e[0] == g[0]
    assert np.array_equal(e[1], g[1]), np.argwhere(e[1] != g[1])[:5]
    assert np.array_equal(e[2], g[2]), np.argwhere(e[2] != g[2])[:5]
    assert np.array_equal(e[3].view(np.uint32), g[3].view(np.uint32))
    assert e[4] == g[4]
    if ctx is not None:
        assert _unsupported(ctx) == n0
    # the large deletions are called precisely, so their consensus alignments (windows beyond 16377 columns) succeeded
    precise = 0
    for s, z in d["truth"]:
        precise += any(v[15] == 2 and v[16] == 1 and abs(int(v[1]) - s) <= 10 and abs(int(v[3]) - (s + z)) <= 10 for v in e[1])
    assert precise >= len(d["truth"]) - 1, (precise, e[1][:, [1, 3, 15, 16]].tolist())


# ---- the whole program on the reference's example --------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("w", [3282, 6500])
def test_example_lr_wide_consensus_window_bcf_identical(tmp_path, w):
    """`delly lr -w W -g ref.fa lr.bam` on the reference's example: the BCF equals the reference's byte for byte and no consensus alignment
    is refused. With dgpu_long_needle alone (the long-read path before dgpu_long_needle_ex) the same runs refused 1 (-w 3282, the smallest
    consensus window that refuses anything on this example; -w 3281 refuses none) and 4 (-w 6500, the most) longNeedle jobs."""
    exe = os.path.join(ROOT, "delly_b200", "bin", "delly_b200")
    assert os.path.exists(DELLY_REF) and os.path.isdir(EX) and os.path.exists(exe)
    ref_out, our_out = str(tmp_path / "ref.bcf"), str(tmp_path / "ours.bcf")
    common = ["-w", str(w), "-g", os.path.join(EX, "ref.fa")]
    _run([DELLY_REF, "lr"] + common + ["-o", ref_out, os.path.join(EX, "lr.bam")])
    r = _run([exe, "lr"] + common + ["-o", our_out, os.path.join(EX, "lr.bam")])
    assert "exceeded a device limit" not in r.stderr, r.stderr[-2000:]
    a, b = _inflate(ref_out), _inflate(our_out)
    assert len(a) > 1000 and a == b, "BCF streams differ"
    assert open(ref_out + ".csi", "rb").read() == open(our_out + ".csi", "rb").read()
