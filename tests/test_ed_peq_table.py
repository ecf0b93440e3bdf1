"""Shared Peq tables of target-sharing HW pairs: every read over one breakpoint is realigned against the same ALT and REF probes, so the
first pair of a key (the ordered pair of probe offsets) to run publishes its Peq table in a per-call hash table, and later pairs of that
key and those lengths copy it instead of building it. Every distance matches the oracle's edlib when many pairs share probes (host,
device and asynchronous forms), when pairs share offsets but not lengths, when the same two probes come in both orders, with N / IUPAC /
lower-case probe bytes, with a probe ending at the arena's last byte, when a call holds more distinct pairs than the table takes, when a
second call reuses the offsets over other bytes, and with empty probes and an odd job count."""
import os

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po

ALPHA = np.frombuffer(b"ACGT", np.uint8)
ODD = np.frombuffer(b"NRYacgtn-", np.uint8)
HW = delly_b200.MODE_HW


def _oracle(b):
    return po.edit_distance_batch(po.oracle(), b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], None, HW,
                                  threads=os.cpu_count() or 1)[0]


def _sites(rng, n_sites, lens, odd=0.0):
    """Per site an ALT and a REF probe (lengths from `lens`, a callable giving two lengths) and the 400 bp of genome they come from."""
    out = []
    for _ in range(n_sites):
        g = ALPHA[rng.integers(0, 4, size=400)]
        la, lr = lens(rng)
        alt = np.concatenate([g[100:100 + la // 2], g[250:250 + la - la // 2]])   # a 150 bp deletion at the breakpoint
        ref = g[100:100 + lr].copy()
        for p in (alt, ref):
            if len(p) and rng.random() < odd:
                pos = rng.integers(0, len(p), size=int(rng.integers(1, 4)))
                p[pos] = ODD[rng.integers(0, len(ODD), size=len(pos))]
        out.append((alt, ref, g))
    return out


def _batch(rng, sites, reads_per_site, swap=0.0, probes_last=False):
    """Jobs 2i / 2i + 1 = (ALT, read) / (REF, read) of one read, reads in shuffled order; with `swap` the pair's probes come in the other
    order for that share of the reads. Probes are stored once per site (reads of a site share their offsets); probes_last puts them after
    the reads, the last probe ending at the arena's last byte."""
    probes, reads, jobs = [], [], []
    for s, (alt, ref, g) in enumerate(sites):
        probes += [alt, ref]
        for _ in range(reads_per_site):
            a0 = int(rng.integers(0, 250))
            reads.append(synth.sub_noise(rng, g[a0:a0 + 150], 0.02))
            pa, pr = 2 * s, 2 * s + 1
            jobs.append((pr, pa) if rng.random() < swap else (pa, pr))
    order = rng.permutation(len(jobs))
    if probes_last:
        arena, off, ln = synth.pack(reads + probes)
        p_off, p_len, r_off = off[len(reads):], ln[len(reads):], off[:len(reads)]
    else:
        arena, off, ln = synth.pack(probes + reads)
        p_off, p_len, r_off = off[:len(probes)], ln[:len(probes)], off[len(probes):]
    q = np.array([jobs[i] for i in order]).reshape(-1)
    t = np.repeat(order, 2)
    return dict(seqs=arena, q_off=p_off[q].copy(), q_len=p_len[q].copy(), t_off=r_off[t].copy(),
                t_len=np.full(len(q), 150, np.uint32))


def _lens_all_classes(rng):
    """two probe lengths of one pair: equal (the benchmark's shape), or any two lengths up to 128"""
    la = int(rng.integers(1, 129))
    return (la, la) if rng.random() < 0.5 else (la, int(rng.integers(1, 129)))


def _dev(b, dev):
    import torch
    t = {n: torch.from_numpy(np.ascontiguousarray(b[n]).view(np.int32)).to(dev) for n in ("q_off", "q_len", "t_off", "t_len")}
    t["seqs"] = torch.from_numpy(np.concatenate([b["seqs"], np.zeros(64, np.uint8)])).to(dev)[:len(b["seqs"])]
    return t


def _run(ctx, b, form="host", bound=None):
    if form == "host":
        return ctx.edit_distance(b["seqs"], b["q_off"], b["q_len"], b["t_off"], b["t_len"], None, HW)
    import torch
    dev = torch.device("cuda", 0)
    t = _dev(b, dev)
    out = torch.full((len(b["q_off"]),), -7, dtype=torch.int32, device=dev)
    if bound:
        assert ctx._lib.dgpu_set_async_bound(ctx.h, bound) == 0
    try:
        ctx.edit_distance_dev(t["seqs"], t["q_off"], t["q_len"], t["t_off"], t["t_len"], None, HW, out, None,
                              torch.cuda.current_stream().cuda_stream)
    finally:
        ctx._lib.dgpu_set_async_bound(ctx.h, 0)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _check(got, b):
    want = _oracle(b)
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, (len(bad), bad[:5], got[bad[:5]], want[bad[:5]], b["q_len"][bad[:5]])


@pytest.mark.gpu
@pytest.mark.parametrize("form,bound", [("host", None), ("dev", None), ("dev", 64), ("dev", 256)])
def test_shared_probes_match_oracle(ctx, form, bound):
    rng = np.random.default_rng(1)
    lens = (lambda r: (int(r.integers(1, 65)),) * 2) if bound == 64 else _lens_all_classes
    b = _batch(rng, _sites(rng, 300, lens), 40, swap=0.1)
    _check(_run(ctx, b, form, bound), b)


@pytest.mark.gpu
def test_same_offsets_other_lengths(ctx):
    """Reads of one site take its probes at one pair of offsets but with lengths cut short by 0..40 bytes, so that pairs with equal keys
    fall into other classes (pair and pack) and must not take each other's tables."""
    rng = np.random.default_rng(2)
    b = _batch(rng, _sites(rng, 200, lambda r: (int(r.integers(41, 129)),) * 2), 30)
    cut = rng.integers(0, 41, size=len(b["q_len"]) // 2)
    b["q_len"][0::2] -= np.minimum(cut, b["q_len"][0::2] - 1).astype(np.uint32)
    b["q_len"][1::2] -= np.minimum(rng.integers(0, 41, size=len(cut)), b["q_len"][1::2] - 1).astype(np.uint32)
    _check(_run(ctx, b), b)


@pytest.mark.gpu
def test_same_probes_both_orders(ctx):
    """Half the reads of a site take (ALT, REF), half (REF, ALT): in a pack slot the order decides which probe is at the bottom."""
    rng = np.random.default_rng(3)
    b = _batch(rng, _sites(rng, 200, lambda r: (int(r.integers(33, 48)), int(r.integers(65, 80)))), 30, swap=0.5)
    _check(_run(ctx, b), b)
    b = _batch(rng, _sites(rng, 200, _lens_all_classes), 30, swap=0.5)
    _check(_run(ctx, b, "dev", 256), b)


@pytest.mark.gpu
def test_probes_with_other_bytes(ctx):
    rng = np.random.default_rng(4)
    b = _batch(rng, _sites(rng, 300, _lens_all_classes, odd=0.5), 20, swap=0.2)
    _check(_run(ctx, b), b)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["host", "dev"])
def test_probe_at_arena_end(ctx, form):
    rng = np.random.default_rng(5)
    for la in (31, 47, 64, 79, 96, 128):
        b = _batch(rng, _sites(rng, 3, lambda r: (la, la)), 20, probes_last=True)
        assert int(b["q_off"].max()) + int(b["q_len"][np.argmax(b["q_off"])]) == len(b["seqs"])
        _check(_run(ctx, b, form), b)


@pytest.mark.gpu
def test_more_pairs_than_the_table(ctx):
    """300 k distinct pairs in one call, more than the 262 k slots of the largest table: pairs that find no slot build their own table."""
    rng = np.random.default_rng(6)
    b = _batch(rng, _sites(rng, 300_000, _lens_all_classes), 1)
    _check(_run(ctx, b, "dev", 256), b)


@pytest.mark.gpu
def test_second_call_other_bytes(ctx):
    """Two calls in a row on one stream over two arenas with the same offsets and other probe bytes: no table outlives its call."""
    import torch
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(7)
    b1 = _batch(rng, _sites(rng, 200, _lens_all_classes), 20)
    b2 = dict(b1)
    b2["seqs"] = b1["seqs"].copy()
    lo = int(b1["q_off"].min())
    hi = int((b1["q_off"].astype(np.int64) + b1["q_len"]).max())
    b2["seqs"][lo:hi] = ALPHA[rng.integers(0, 4, size=hi - lo)]
    t1, t2 = _dev(b1, dev), _dev(b2, dev)
    o1 = torch.full((len(b1["q_off"]),), -7, dtype=torch.int32, device=dev)
    o2 = torch.full_like(o1, -7)
    st = torch.cuda.current_stream().cuda_stream
    assert ctx._lib.dgpu_set_async_bound(ctx.h, 256) == 0
    try:
        for t, o in ((t1, o1), (t2, o2)):
            ctx.edit_distance_dev(t["seqs"], t["q_off"], t["q_len"], t["t_off"], t["t_len"], None, HW, o, None, st)
    finally:
        ctx._lib.dgpu_set_async_bound(ctx.h, 0)
    torch.cuda.synchronize()
    _check(o1.cpu().numpy(), b1)
    _check(o2.cpu().numpy(), b2)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["host", "dev"])
def test_empty_probes_and_odd_n(ctx, form):
    rng = np.random.default_rng(8)
    b = _batch(rng, _sites(rng, 100, lambda r: (int(r.integers(0, 3)) * int(r.integers(1, 129)), int(r.integers(1, 129)))), 20)
    b = {k: (v[:-1] if k != "seqs" else v) for k, v in b.items()}
    assert len(b["q_off"]) % 2 == 1 and (b["q_len"] == 0).any()
    _check(_run(ctx, b, form), b)


def test_batches_share_probes():
    """CPU check of the generator: reads of a site share their probes' offsets, so the pairs repeat."""
    rng = np.random.default_rng(9)
    b = _batch(rng, _sites(rng, 50, _lens_all_classes), 10, swap=0.5)
    keys = set(zip(b["q_off"][0::2].tolist(), b["q_off"][1::2].tolist()))
    assert len(keys) <= 100 and len(b["q_off"]) == 1000
    assert (b["t_off"][0::2] == b["t_off"][1::2]).all()
