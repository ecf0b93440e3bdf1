"""Edit paths over aligned target slices wider than 16384 columns (dgpu_edit_path_wide): NW, HW and SHW slices of 16385 columns up to
DGPU_EP_MAX_SLICE, thin wide Hirschberg leaves on both sides of the split rule, shared-arena layouts, batches mixing ordinary and wide jobs,
the device form, the max_slice checks and the edlib C API, each path compared op for op with the reference's edlib and replayed against its
sequences. Then the long-read chain with 7-25 kb insertions, whose consensus rounds send windows of more than 16384 bases through edit
paths, against the reference's chain (GPU, and on the CPU through the test stand-in)."""
import ctypes as C
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po
from test_edit_path_long import EQS, IUPAC_EQ, _batch, _noisy, _packed, _rand, _replay, _seq, _sprinkle
from test_edlib_compat import Pair, _bind
from test_host_genotype import LR_CFG
from test_host_split import _p
from test_msa_large import _build_standin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = delly_b200.EP_MAX_SLICE
THREADS = os.cpu_count() or 1


def _ref_paths(ref, b, mode, eq, task=None):
    """The reference's (dist, end, start, ops) per job, the jobs spread over host threads (ctypes releases the GIL)."""
    n = len(b["q_off"])
    tasks = task if task is not None else [2] * n
    with ThreadPoolExecutor(THREADS) as ex:
        return list(ex.map(lambda i: po.edit_distance(ref, _seq(b, i, "q"), _seq(b, i, "t"), -1, mode, task=tasks[i], eq=eq), range(n)))


def _check(ctx, ref, b, mode, eq, max_slice=CAP, status=None):
    """dgpu_edit_path_wide against the reference's edlib on every job: distance, locations, status and ops; the traced paths are replayed.
    A job with expected status 2 must carry the reference's distance and locations and no ops. Returns the device's results."""
    n = len(b["q_off"])
    want = np.zeros(n, np.uint32) if status is None else np.asarray(status, np.uint32)
    res = ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], mode, eq=eq, max_slice=max_slice)
    d, st, en, ops, stat = res
    refs = _ref_paths(ref, b, mode, eq, [1 if w == 2 else 2 for w in want])
    bad = []
    for i, (rd, re, rs, rops) in enumerate(refs):
        if (d[i], st[i], en[i], stat[i]) != (rd, rs, re, want[i]) or ops[i] != (b"" if want[i] == 2 else rops):
            bad.append((i, int(b["q_len"][i]), int(b["t_len"][i]), int(stat[i]), int(d[i]), int(st[i]), int(en[i]), len(ops[i]), "ref", rd, rs, re, len(rops)))
    assert not bad, (mode, bad[:6])
    for i in range(n):
        if want[i] == 0:
            _replay(_seq(b, i, "q"), _seq(b, i, "t"), int(d[i]), int(st[i]), int(en[i]), ops[i], eq)
    return res


def _slices(res):
    _, st, en, _, _ = res
    return [int(e) - int(s) + 1 for s, e in zip(st, en)]


# ---------------------------------------------------------------------------------------------------------------------------------------
# NW slices, near the cap, HW / SHW in the msaWfa shape

NW_SIMILAR = [16385, 16448, 20000, 32768, 32769, 40000, 65535]
NW_UNRELATED = [16385, 20000, 32769, 40000]


def _nw_batch(eq, seed):
    """NW pairs of each width: 5-12 % substitutions plus indels (band classes certify their segments near the leaves only), and unrelated
    pairs (no band class: the half columns of a pair wider than 32768 reach seg_half_wide_kernel at the top level)."""
    rng = np.random.default_rng(seed)
    seqs = []
    for i, L in enumerate(NW_SIMILAR):
        t = _rand(rng, L)
        seqs += [_noisy(rng, t, 0.05 + 0.07 * i / (len(NW_SIMILAR) - 1)), _sprinkle(rng, t) if eq else t]
    for L in NW_UNRELATED + ([] if eq else [65535]):
        seqs += [_rand(rng, L - int(rng.integers(0, 600))), _rand(rng, L)]
    return _packed(seqs)


@pytest.mark.gpu
@EQS
def test_wide_nw_slices(ctx, ref, eq):
    """NW slices of 16385-65535 columns, similar and unrelated pairs, with and without the 20 IUPAC pairs."""
    b = _nw_batch(eq, 3100 + len(eq))
    res = _check(ctx, ref, b, 0, eq)
    assert set(NW_SIMILAR) <= set(_slices(res))


@pytest.mark.gpu
def test_wide_nw_near_cap(ctx, ref):
    """A slice a few columns under DGPU_EP_MAX_SLICE (8 % divergence) and one of exactly the cap."""
    rng = np.random.default_rng(3200)
    seqs = []
    for L in (CAP - 37, CAP):
        t = _rand(rng, L)
        seqs += [_noisy(rng, t, 0.08 if L < CAP else 0.03), t]
    res = _check(ctx, ref, _packed(seqs), 0, b"")
    assert _slices(res) == [CAP - 37, CAP]


def _msawfa_batch(mode, seed, n=4):
    """msaWfa's HW call at long-read sizes: a read of 17-40 kb (ONT-like: 4 % substitutions, 3 % insertions, 3 % deletions) against a
    gapped IUPAC consensus of 20-60 kb that contains it (SHW: the read starts at the consensus' first base)."""
    rng = np.random.default_rng(seed)
    seqs = []
    for _ in range(n):
        R = int(rng.integers(17_000, 40_001))
        T = int(rng.integers(max(20_000, R + 500), 60_001))
        base = _rand(rng, T)
        a = 0 if mode == 1 else int(rng.integers(0, T - R + 1))
        read = synth.mutate_fast(rng, base[a:a + R], sub=0.04, ins=0.03, dele=0.03)
        cons = _sprinkle(rng, base, 0.03)
        gaps = np.sort(rng.choice(T, size=T // 30, replace=False))
        seqs += [read, np.insert(cons, gaps, np.uint8(ord("-")))]
    return _packed(seqs)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 2], ids=["shw", "hw"])
def test_wide_msawfa_shape(ctx, ref, mode):
    """HW and SHW paths of 17-40 kb reads against 20-60 kb gapped IUPAC consensus strings with the 20 pairs."""
    b = _msawfa_batch(mode, 3300 + mode)
    res = _check(ctx, ref, b, mode, IUPAC_EQ)
    assert max(_slices(res)) > 16384


# ---------------------------------------------------------------------------------------------------------------------------------------
# thin wide leaves: at most two 64-row blocks, more than 16384 columns

LEAF_TARGETS = {1: (16385, 30000, 37449, 37450), 63: (16385, 37449, 37450), 64: (20000, 37449, 37450), 65: (16385, 21845, 21846),
                127: (18000, 21845, 21846), 128: (16385, 21845, 21846)}


def _leaf(m, n):
    return 20 * ((m + 63) // 64) * n + 8 * n < 1 << 20


@pytest.mark.gpu
@EQS
def test_wide_thin_leaves(ctx, ref, eq):
    """NW queries of 1-128 bases against targets of 16385-37450 bases, on both sides of the split rule (37449 / 37450 for m <= 64,
    21845 / 21846 for 64 < m <= 128): unrelated queries and queries taken from inside their target."""
    rng = np.random.default_rng(3400 + len(eq))
    seqs = []
    for m, ns in LEAF_TARGETS.items():
        for n in ns:
            t = _rand(rng, n)
            tt = _sprinkle(rng, t) if eq else t
            a = int(rng.integers(0, n - m))
            seqs += [_rand(rng, m), tt, t[a:a + m].copy(), tt]
    b = _packed(seqs)
    _check(ctx, ref, b, 0, eq)
    ml = zip(b["q_len"].tolist(), b["t_len"].tolist())
    assert sum(_leaf(m, n) and n > 16384 for m, n in ml) >= 24


# ---------------------------------------------------------------------------------------------------------------------------------------
# shared arena bytes, mixed batches, the device form

def _wide_shared_arena(seed):
    """A 120 kb contig; queries inside their own targets, a query equal to its target, overlapping windows of the contig, and a window that
    is the query of one job and the target of another, all with slices wider than 16384 columns."""
    rng = np.random.default_rng(seed)
    C_ = 120_000
    contig = _rand(rng, C_)
    jobs = []
    for tl, a, ql in ((40_000, 9_000, 20_000), (30_000, 0, 17_000), (25_000, 3_000, 22_000)):
        o = int(rng.integers(0, C_ - tl))
        jobs.append((o + a, ql, o, tl))
    o = int(rng.integers(0, C_ - 18_000))
    jobs.append((o, 18_000, o, 18_000))
    w = [(10_000, 30_000), (25_000, 30_000), (38_000, 26_000)]
    for (o1, l1), (o2, l2) in zip(w, w[1:]):
        jobs.append((o1, l1, o2, l2))
    read = synth.mutate_fast(rng, contig[50_000:70_000], sub=0.03, ins=0.01, dele=0.01)
    jobs.append((C_, len(read), 45_000, 30_000))
    return _batch(np.concatenate([contig, read]), jobs)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_wide_shared_arena_bytes(ctx, ref, mode):
    """Sequences that share arena bytes, at slices wider than 16384 columns, in every mode."""
    res = _check(ctx, ref, _wide_shared_arena(3500), mode, b"")
    assert max(_slices(res)) > 16384


def _mixed_batch(seed):
    """Ordinary NW jobs (slices of 50 bases to 16384 columns) interleaved with wide ones."""
    rng = np.random.default_rng(seed)
    seqs, wide = [], []
    for L in (50, 900, 4000, 16384, 17000, 300, 12000, 33000, 2500, 16384, 25000, 700):
        t = _rand(rng, L)
        q = synth.mutate_fast(rng, t, sub=0.04, ins=0.02, dele=0.02) if L % 2 == 0 else _rand(rng, max(1, L - 200))
        seqs += [q, t]
        wide.append(L > 16384)
    return _packed(seqs), np.array(wide)


@pytest.mark.gpu
def test_wide_mixed_batch_keeps_ordinary_jobs(ctx, ref):
    """A batch mixing ordinary and wide jobs: every job matches the reference, and the ordinary jobs are byte-identical to what
    dgpu_edit_path_ex gives for the same batch (where the wide jobs get status 2)."""
    b, wide = _mixed_batch(3600)
    res = _check(ctx, ref, b, 0, b"")
    old = ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], 0)
    assert (old[4][wide] == 2).all() and (old[4][~wide] == 0).all()
    for k in range(3):
        assert np.array_equal(old[k][~wide], res[k][~wide])
    assert all(old[3][i] == res[3][i] for i in np.nonzero(~wide)[0])


@pytest.mark.gpu
def test_wide_device_form_on_a_side_stream(ctx):
    """dgpu_edit_path_wide_dev on a non-default stream gives the host form's results."""
    import torch
    b = _nw_batch(IUPAC_EQ, 3700)
    host = ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], 0, eq=IUPAC_EQ, max_slice=CAP)
    n = len(b["q_off"])
    cap = b["q_len"].astype(np.uint64) + b["t_len"].astype(np.uint64)
    ops_off = np.concatenate([[0], np.cumsum(cap)[:-1]]).astype(np.uint64)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int32 if a.dtype.itemsize == 4 else a.dtype)).cuda()
    arena = np.zeros((len(b["seqs"]) + 64 + 15) // 16 * 16, np.uint8)
    arena[:len(b["seqs"])] = b["seqs"]
    seqs = torch.from_numpy(arena).cuda()
    qo, ql, to, tl = (dev(b[k]) for k in ("q_off", "q_len", "t_off", "t_len"))
    oo = torch.from_numpy(ops_off.view(np.int64)).cuda()
    out = [torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(5)]
    ops = torch.zeros(int(cap.sum()) + 64, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ctx.edit_path_dev(seqs, qo, ql, to, tl, 0, out[0], out[1], out[2], ops, oo, out[3], out[4], eq=IUPAC_EQ, stream=s.cuda_stream, max_slice=CAP)
    s.synchronize()
    d, st, en, ol, stat = (o.cpu().numpy() for o in out)
    assert np.array_equal(d, host[0]) and np.array_equal(st, host[1]) and np.array_equal(en, host[2]) and not stat.any()
    o = ops.cpu().numpy()
    assert all(o[int(ops_off[i]):int(ops_off[i]) + int(ol[i])].tobytes() == host[3][i] for i in range(n))


# ---------------------------------------------------------------------------------------------------------------------------------------
# max_slice

@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])
def test_wide_max_slice(ctx, ref, mode):
    """A job one column over max_slice gets status 2 alone and keeps the reference's distance and locations; max_slice = 0 and
    DGPU_EP_MAX_SLICE + 1 are argument errors of both forms."""
    rng = np.random.default_rng(3800 + mode)
    seqs = []
    for L in (20_000, 20_001, 3000, 19_999):
        t = _rand(rng, L + (3000 if mode == 2 else 0))
        a = 1500 if mode == 2 else 0
        seqs += [_noisy(rng, t[a:a + L], 0.03), t]
    b = _packed(seqs)
    res = _check(ctx, ref, b, mode, b"", max_slice=20_000, status=[0, 2, 0, 0])
    assert _slices(res) == [20_000, 20_001, 3000, 19_999]
    lib = delly_b200.lib()
    for bad in (0, CAP + 1):
        with pytest.raises(delly_b200.DgpuError, match="max_slice"):
            ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], mode, max_slice=bad)
        z = C.c_void_p(0)
        rc = lib.dgpu_edit_path_wide_dev(ctx.h, z, C.c_uint64(0), z, z, z, z, mode, None, C.c_uint32(0), C.c_uint64(1), z, z, z, z, z, z, z,
                                         C.c_uint32(bad), z)
        assert rc == -2


def _tall_batch(seed):
    """NW pairs whose query holds a 225 kb insertion: the top-level half columns have about 241 k rows, more than seg_kernel can stage in
    shared memory, while the leaves below them (about 225 k rows, at most 14 columns) still fit it."""
    rng = np.random.default_rng(seed)
    seqs = []
    for n in (16_000, 20_000):
        t = _rand(rng, n)
        h = n // 2
        seqs += [np.concatenate([_noisy(rng, t[:h], 0.03), _rand(rng, 225_000), _noisy(rng, t[h:], 0.03)]), t]
    return _packed(seqs)


@pytest.mark.gpu
def test_tall_half_columns(ctx, ref):
    """Half columns with more rows than seg_kernel's shared memory holds run on seg_half_wide_kernel in every form: through
    dgpu_edit_path_ex the 16000-column job is traced (such a call used to fail with a CUDA error) and the 20000-column one gets status 2;
    through dgpu_edit_path_wide both are traced. Every path matches the reference's."""
    b = _tall_batch(3950)
    assert (b["q_len"] > 240_000).all()
    res = _check(ctx, ref, b, 0, b"")
    old = _check(ctx, ref, b, 0, b"", max_slice=16384, status=[0, 2])
    assert old[3][0] == res[3][0]
    classic = ctx.edit_path(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], 0)
    assert list(classic[4]) == [0, 2] and classic[3][0] == res[3][0] and classic[0][1] == res[0][1]


@pytest.mark.gpu
def test_wide_slices_without_band_passes():
    """The NW, leaf, msaWfa and mixed batches once more with DGPU_EP_NO_BAND=1 (read once per process): no band class, so the wide
    segments all go through seg_half_wide_kernel / seg_leaf_wide_kernel. They run in a child pytest that has exited when this test returns."""
    if os.environ.get("DGPU_EP_NO_BAND"):
        pytest.skip("this is the child run")
    env = dict(os.environ, DGPU_EP_NO_BAND="1")
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", "-k",
           "wide_nw_slices or thin_leaves or msawfa_shape or mixed_batch or shared_arena or tall_half", os.path.abspath(__file__)]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout, r.stdout[-2000:]


# ---------------------------------------------------------------------------------------------------------------------------------------
# the host mirrors: the edlib C API and the long-read chain

@pytest.fixture(params=[pytest.param("gpu", marks=pytest.mark.gpu), "edlib-standin"])
def hostdev_epw(request, ref):
    """(host library, context handle): the real libraries on an H100, or the CPU stand-in with dgpu_edit_path_wide forwarded to the
    reference's edlib"""
    if request.param == "gpu":
        return delly_b200.hostlib(), request.getfixturevalue("ctx").h
    lib = C.CDLL(_build_standin("libhost_standin_edit_path_wide.so", ["host_standin.cpp", "edit_path_wide_standin.cpp"], shared=True))
    lib.standin_ctx.restype = C.c_void_p
    return lib, C.c_void_p(lib.standin_ctx())


def test_wide_edlib_align_path(hostdev_epw, ref):
    """edlibAlign(..., EDLIB_TASK_PATH) through include/dgpu_edlib.h on 20-40 kb pairs, with and without equalities: the reference's
    distance, locations, alignment and CIGAR."""
    H, _ = hostdev_epw
    _bind(H)
    if hasattr(H, "standin_edlib_compat_init"):
        H.standin_edlib_compat_init()
    H.dgpu_edlibAlignmentToCigar.restype = C.c_void_p
    libc = C.CDLL(None)
    libc.free.argtypes = [C.c_void_p]
    rng = np.random.default_rng(3900)
    for i, (R, T, mode) in enumerate(((20_000, 20_000, 0), (25_000, 38_000, 2), (30_000, 40_000, 1), (40_000, 40_000, 0))):
        t = _rand(rng, T)
        q = synth.mutate_fast(rng, t[:R], sub=0.03, ins=0.01, dele=0.01) if mode == 1 else _noisy(rng, t[T - R:] if mode == 2 else t[:R], 0.04)
        eq = b"NANCNGNT" if i % 2 else b""
        if eq:
            q = q.copy(); q[rng.integers(0, len(q), size=50)] = ord("N")
        pairs = (Pair * max(1, len(eq) // 2))()
        for j in range(len(eq) // 2):
            pairs[j].first = eq[2 * j:2 * j + 1]; pairs[j].second = eq[2 * j + 1:2 * j + 2]
        qb, tb = bytes(q), bytes(t)
        d, e, s, ops = po.edit_distance(ref, qb, tb, k=-1, mode=mode, task=2, eq=eq)
        r = H.dgpu_edlibAlign(qb, len(qb), tb, len(tb), H.dgpu_edlibNewAlignConfig(-1, mode, 2, pairs if eq else None, len(eq) // 2))
        try:
            assert r.status == 0 and r.editDistance == d and r.endLocations[0] == e and r.startLocations[0] == s, (i, r.editDistance, d)
            assert e - s + 1 > 16384
            got = bytes(r.alignment[:r.alignmentLength])
            assert got == ops, i
            out = C.create_string_buffer(2 * len(ops) + 8)
            assert ref.ref_edlib_cigar(ops, len(ops), 1, out, len(out)) >= 0
            cg = H.dgpu_edlibAlignmentToCigar(got, len(got), 1)
            assert C.string_at(cg) == out.value
            libc.free(cg)
        finally:
            H.dgpu_edlibFreeAlignResult(r)


INS_SIZES = (7500, 12000, 18500, 25000)


def _simulate_lr_large_ins(seed, sizes=INS_SIZES, cov=12, zyg=(1, 2, 2, 2)):
    """A diploid sample with large heterozygous / homozygous insertions of random sequence on contig 0, sequenced with 18-50 kb reads with
    5 % substitutions; a read over an insertion carries it as an I operation of its CIGAR (as _simulate_lr_large_dels builds deletions)."""
    rng = np.random.default_rng(seed)
    L0 = 60000 + 70000 * len(sizes)
    ref0 = synth._ACGT[rng.integers(0, 4, size=L0, dtype=np.uint8)]; ref1 = synth._ACGT[rng.integers(0, 4, size=20000, dtype=np.uint8)]
    starts = [40000 + 70000 * i + int(rng.integers(0, 2000)) for i in range(len(sizes))]
    inserts = [synth._ACGT[rng.integers(0, 4, size=z, dtype=np.uint8)] for z in sizes]
    recs, cigs, reads = [], [], []
    total = int(L0 * cov / 34000)
    for rid in range(total):
        tid = 0 if rng.random() < 0.95 else 1
        L = int(rng.integers(18000, 50001)) if tid == 0 else int(rng.integers(3000, 8000))
        hap = int(rng.integers(0, 2))
        G = ref0 if tid == 0 else ref1
        p = int(rng.integers(0, len(G) - L - 2000))
        ops, seq, rp, left = [], [], p, L
        ev = [(s, i) for i, (s, g) in enumerate(zip(starts, zyg)) if tid == 0 and (g == 2 or hap == 1) and s > p + 300]
        for s, i in ev:
            z = sizes[i]
            if s - rp + z >= left - 1500:
                break
            ops.append((0, s - rp)); seq.append(G[rp:s]); left -= s - rp; rp = s
            ops.append((1, z)); seq.append(inserts[i]); left -= z
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


CONS_W = 65536


def test_delly_lr_call_large_insertions_match_reference(hostdev_epw, ref5):
    """`delly lr -i 40000` on insertions of 7.5-25 kb spanned by 18-50 kb reads: the consensus rounds align read windows of more than
    16384 bases. Every record field, the consensus strings and the GL bit patterns equal the reference's, the insertions are called
    precise, and no edit-path job is refused."""
    H, ctxh = hostdev_epw
    H.dh_path_jobs_refused.restype = C.c_uint64
    d = _simulate_lr_large_ins(2026)
    nrec = len(d["rec"])
    cfg = LR_CFG.copy()
    cfg[8] = 40000   # indelsize
    ref5.ref_hash_lr_name5.restype = C.c_uint64
    seeds = np.array([ref5.ref_hash_lr_name5(f"q{int(r[11])}".encode()) for r in d["rec"]], np.uint64)
    refused0 = H.dh_path_jobs_refused()
    outs = []
    for which in ("ref", "ours"):
        sv = np.zeros((512, 20), np.int32); fmt = np.zeros((512, 14), np.int32); gl = np.zeros((512, 3), np.float32)
        co = np.zeros((512, CONS_W), np.uint8); cl = np.zeros(512, np.int32)
        tail = (_p(d["cig"]), _p(d["reads"]), _p(cfg), C.c_float(0.9), C.c_float(0.5), _p(sv), 512, _p(fmt), _p(gl), _p(co), CONS_W, _p(cl))
        if which == "ref":
            n = ref5.ref_delly_lr_call(_p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 2, _p(d["rec"]), nrec, *tail)
        else:
            n = H.dh_delly_lr_call(ctxh, _p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 2, _p(d["rec"]), _p(seeds), nrec, *tail)
        assert n > 0, n
        outs.append((n, sv[:n].copy(), fmt[:n].copy(), gl[:n].copy(), [co[i, :cl[i]].tobytes() for i in range(n)]))
    e, g = outs
    assert e[0] == g[0], (e[0], g[0])
    assert np.array_equal(e[1], g[1]), np.argwhere(e[1] != g[1])[:5]
    assert np.array_equal(e[2], g[2]), np.argwhere(e[2] != g[2])[:5]
    assert np.array_equal(e[3].view(np.uint32), g[3].view(np.uint32))
    assert e[4] == g[4], [i for i in range(e[0]) if e[4][i] != g[4][i]]
    assert H.dh_path_jobs_refused() == refused0
    precise = [any(v[15] == 4 and v[16] == 1 and abs(int(v[1]) - s) <= 30 and abs(int(v[13]) - z) <= 0.05 * z for v in e[1]) for s, z in d["truth"]]
    assert all(precise), (precise, e[1][:, [1, 3, 13, 15, 16]].tolist())
    assert max(len(c) for c in e[4]) > 16384


def test_delly_lr_call_full_chain_large_insertion(hostdev_epw, ref9, ref8):
    """The complete long-read chain (annotation, MM / ML methylation) with insertions of 17-25 kb: the methylation placement aligns each
    read's insertion against the consensus insertion, slices of more than 16384 columns. Every output equals the reference's."""
    from test_methyl import _with_tags
    from test_svanno import _templates
    H, ctxh = hostdev_epw
    H.dh_path_jobs_refused.restype = C.c_uint64
    _, tpl_arena, tpl_off = _templates(ref8)
    d = _with_tags(_simulate_lr_large_ins(2027, sizes=(17500, 25000), cov=10, zyg=(2, 1)), 98)
    nrec = len(d["rec"])
    cfg = LR_CFG.copy()
    cfg[8] = 40000
    ref9.ref_hash_lr_name5.restype = C.c_uint64
    seeds = np.array([ref9.ref_hash_lr_name5(f"q{int(r[11])}".encode()) for r in d["rec"]], np.uint64)
    refused0 = H.dh_path_jobs_refused()
    outs = []
    for which in ("ref", "ours"):
        sv = np.zeros((512, 20), np.int32); fmt = np.zeros((512, 14), np.int32); gl = np.zeros((512, 3), np.float32)
        co = np.zeros((512, CONS_W), np.uint8); cl = np.zeros(512, np.int32)
        an = np.full((512, 5), -9, np.int32); me = np.full((512, 16), -9, np.int32); al = np.zeros((512, CONS_W), np.uint8); all_ = np.zeros(512, np.int32)
        head = (_p(d["cig"]), _p(d["reads"]), _p(cfg), C.c_float(0.9), C.c_float(0.5), _p(sv), 512, _p(fmt), _p(gl), _p(co), CONS_W, _p(cl), _p(d["tagflags"]),
                _p(d["mm"]), _p(d["mm_off"]), _p(d["ml"]), _p(d["ml_off"]), 400, 128, 1)
        tail = (C.c_float(0.8), C.c_float(0.85), _p(an), _p(me), _p(al), CONS_W, _p(all_))
        if which == "ref":
            n = ref9.ref_delly_lr_call_ex(_p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 2, _p(d["rec"]), nrec, *head, *tail)
        else:
            n = H.dh_delly_lr_call_ex(ctxh, _p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 2, _p(d["rec"]), _p(seeds), nrec, *head, _p(tpl_arena), _p(tpl_off), *tail)
        assert n > 0, n
        outs.append((n, sv[:n].copy(), fmt[:n].copy(), gl[:n].copy(), [co[i, :cl[i]].tobytes() for i in range(n)], an[:n].copy(), me[:n].copy(),
                     [al[i, :all_[i]].tobytes() for i in range(n)]))
    e, g = outs
    assert e[0] == g[0]
    assert np.array_equal(e[1], g[1]), np.argwhere(e[1] != g[1])[:5]
    assert np.array_equal(e[2], g[2]), np.argwhere(e[2] != g[2])[:5]
    assert np.array_equal(e[3].view(np.uint32), g[3].view(np.uint32))
    assert e[4] == g[4] and e[7] == g[7]
    assert np.array_equal(e[5], g[5]) and np.array_equal(e[6], g[6])
    assert H.dh_path_jobs_refused() == refused0
    ins = [v for v in e[1] if v[15] == 4 and v[16] == 1 and v[13] > 16384]
    assert ins, e[1][:, [1, 13, 15, 16]].tolist()
