"""ed_pack_kernel: the two HW jobs of a pair (jobs 2i and 2i + 1 on one target, no end locations) share one column of 3 or 5 words when
their queries fit it (pack_fits: A of 33-63 bp with B of up to 95 - |A| bp, or A of 65-95 bp with B of up to 159 - |A|, in either job
order). Every job's distance matches the oracle's edlib for every such length pair, pairs just outside the bounds do not pack, and the pack
kernels run in the asynchronous device form and in every range of the pipelined host form."""
import os

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po

ALPHA = np.frombuffer(b"ACGT", np.uint8)
ODD = np.frombuffer(b"NRYacgtn-", np.uint8)
TLENS = list(range(140, 156)) + [1, 2, 5, 17, 31, 46, 63, 64, 100, 297, 300]
PACKS = ((3, 1), (5, 2))


def pack_fits(ma, mb, w, wa):
    return (ma > 32 * wa) & (ma <= 32 * wa + 31) & (mb >= 1) & (ma + mb < 32 * w)


def pack_class(m0, m1):
    """The W of the pack class of jobs with query lengths m0 (job 2i) and m1 (job 2i + 1), or 0."""
    for w, wa in PACKS:
        if pack_fits(m0, m1, w, wa) or pack_fits(m1, m0, w, wa):
            return w
    return 0


def _odd(rng, a, rate):
    a = a.copy()
    if len(a) and rng.random() < rate:
        pos = rng.integers(0, len(a), size=int(rng.integers(1, 4)))
        a[pos] = ODD[rng.integers(0, len(ODD), size=len(pos))]
    return a


def _batch(seed, lens):
    """One target per (m0, m1) in `lens`, jobs 2i / 2i + 1 = the two probes on it: probes cut from the target with noise or random, N /
    IUPAC / lower-case bytes in probes and targets, targets of lengths of every residue mod 16."""
    rng = np.random.default_rng(seed)
    seqs, jobs = [], []
    for i, (m0, m1) in enumerate(lens):
        tl = TLENS[i % len(TLENS)] if rng.random() < 0.8 else int(rng.integers(1, 200))
        t = ALPHA[rng.integers(0, 4, size=tl)]
        qs = []
        for ql in (m0, m1):
            if rng.random() < 0.7 and tl >= ql:
                a0 = int(rng.integers(0, tl - ql + 1))
                q = synth.sub_noise(rng, t[a0:a0 + ql], 0.05)
            else:
                q = ALPHA[rng.integers(0, 4, size=ql)]
            qs.append(_odd(rng, q, 0.2))
        t = _odd(rng, t, 0.3)
        ti = len(seqs)
        seqs.append(t)
        for q in qs:
            seqs.append(q)
            jobs.append((len(seqs) - 1, ti))
    arena, off, ln = synth.pack(seqs)
    qi = np.array([j[0] for j in jobs]); ti = np.array([j[1] for j in jobs])
    return dict(seqs=arena, q_off=off[qi].copy(), q_len=ln[qi].copy(), t_off=off[ti].copy(), t_len=ln[ti].copy())


def _fitting_lens():
    """Every (mA, mB) that fits a pack class in the order (mA, mB), in both job orders."""
    lens = [(ma, mb) for ma in range(33, 64) for mb in range(1, 96 - ma)]
    lens += [(ma, mb) for ma in range(65, 96) for mb in range(1, 160 - ma)]
    return lens + [(mb, ma) for ma, mb in lens]


def _outside_lens():
    """Pairs just outside the bounds: A's last row in the word above WA (64, 96), one row too many for a separator, partners past 128."""
    lens = [(64, mb) for mb in (1, 31, 32, 33, 63, 64)] + [(96, mb) for mb in (1, 32, 63, 64)]
    lens += [(ma, 96 - ma) for ma in range(33, 64)] + [(ma, 160 - ma) for ma in range(65, 96)]
    lens += [(ma, 129) for ma in (33, 63, 65, 95)] + [(32, 32), (31, 64), (16, 96)]
    return lens + [(mb, ma) for ma, mb in lens]


def _ks(rng, d):
    sel = rng.integers(0, 4, size=len(d))
    return np.where(sel == 0, d - 1, np.where(sel == 1, d, np.where(sel == 2, d + 1, -1))).astype(np.int32)


def _oracle(b, k):
    return po.edit_distance_batch(po.oracle(), b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, 2,
                                  threads=os.cpu_count() or 1)[0]


def _pack_launches(prof):
    return sum(e.count for e in prof.key_averages() if "ed_pack_kernel" in e.key)


def test_length_sets_cover_the_bounds():
    fit = _fitting_lens()
    assert all(pack_class(m0, m1) for m0, m1 in fit)
    assert {pack_class(m0, m1) for m0, m1 in fit} == {3, 5}
    assert (33, 62) in fit and (62, 33) in fit and (95, 64) in fit and (64, 95) in fit and (63, 1) in fit and (1, 63) in fit
    assert not any(pack_class(m0, m1) for m0, m1 in _outside_lens())
    b = _batch(1, fit[:200])
    assert {int(x) % 16 for x in b["t_len"]} == set(range(16))


@pytest.mark.gpu
def test_every_fitting_length_pair_matches_oracle(ctx):
    import torch
    from torch.profiler import ProfilerActivity, profile
    b = _batch(2, _fitting_lens())
    k = _ks(np.random.default_rng(3), _oracle(b, None))
    d = _oracle(b, k)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, delly_b200.MODE_HW)
        torch.cuda.synchronize()
    bad = np.nonzero(g != d)[0]
    assert len(bad) == 0, (bad[:5], g[bad[:5]], d[bad[:5]], b["q_len"][bad[:5]], b["q_len"][bad[:5] ^ 1], b["t_len"][bad[:5]])
    assert _pack_launches(prof) == 2
    # the same jobs with end locations take the other kernels and give the same distances
    ge, _ = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, delly_b200.MODE_HW, want_end=True)
    assert np.array_equal(ge, g)


@pytest.mark.gpu
def test_pairs_outside_the_bounds_do_not_pack(ctx):
    import torch
    from torch.profiler import ProfilerActivity, profile
    b = _batch(4, _outside_lens())
    k = _ks(np.random.default_rng(5), _oracle(b, None))
    d = _oracle(b, k)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], k, delly_b200.MODE_HW)
        torch.cuda.synchronize()
    assert _pack_launches(prof) == 0
    assert np.array_equal(g, d)


@pytest.mark.gpu
@pytest.mark.parametrize("bound", [64, 256])
def test_pack_in_async_device_form(ctx, bound):
    """dgpu_set_async_bound: the pack grids are sized from n / 2, the 5-word class only launched for bounds above 64."""
    import torch
    lens = [lp for lp in _fitting_lens() if max(lp) <= bound]
    b = _batch(6, lens)
    k = _ks(np.random.default_rng(7), _oracle(b, None))
    d = _oracle(b, k)
    dev = torch.device("cuda", 0)
    t = {n: torch.from_numpy(np.ascontiguousarray(b[n]).view(np.int32) if n != "seqs" else b[n]).to(dev)
         for n in ("seqs", "q_off", "q_len", "t_off", "t_len")}
    kt = torch.from_numpy(k).to(dev)
    out = torch.full((len(k),), -7, dtype=torch.int32, device=dev)
    lib = ctx._lib
    assert lib.dgpu_set_async_bound(ctx.h, bound) == 0
    try:
        ctx.edit_distance_dev(t["seqs"], t["q_off"], t["q_len"], t["t_off"], t["t_len"], kt, delly_b200.MODE_HW, out, None, None)
        torch.cuda.synchronize()
    finally:
        lib.dgpu_set_async_bound(ctx.h, 0)
    assert np.array_equal(out.cpu().numpy(), d)


@pytest.mark.gpu
def test_pipelined_host_form_packs_in_every_range(ctx):
    """3 * 2^18 - 2 genotyping jobs in two ranges: both pack kernels run in both, and the distances match the oracle."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    n = 3 * (1 << 18) - 2
    b = synth.k1_genotype_batch(n, seed=33)
    assert len(b["seqs"]) >= 32 << 20
    d = _oracle(b, b["k"])
    i = np.arange(0, n, 2)
    shared = (b["t_off"][i] == b["t_off"][i + 1]) & (b["t_len"][i] == b["t_len"][i + 1])
    w = np.array([pack_class(int(x), int(y)) for x, y in zip(b["q_len"][i], b["q_len"][i + 1])]) * shared
    jobs_per = 393216
    want = len(set(w[(i < jobs_per) & (w > 0)].tolist())) + len(set(w[(i >= jobs_per) & (w > 0)].tolist()))
    assert want == 4
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g = ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], b["k"], delly_b200.MODE_HW)
        torch.cuda.synchronize()
    assert _pack_launches(prof) == want
    assert np.array_equal(g, d)
