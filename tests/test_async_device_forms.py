"""The asynchronous device forms of longNeedle and the MSA (include/dgpu.h: dgpu_set_ln_async_bound, dgpu_set_msa_async_bound).

Under a bound the device forms read nothing back: longNeedle plans its workspace on the device. Checked here: byte-identical results to the
synchronous device form and the oracle (sr, lr, IUPAC and wide shapes, and one call mixing them), calls that return while the device is still
busy, an MSA -> longNeedle chain captured into a CUDA graph and replayed on new data (two contexts on one device), refusals of jobs beyond the
bound, and the synchronous forms unchanged after switching back."""
import ctypes as C
import os
import re
import time

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po
from test_long_needle import _edge_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("dgpu_set_ln_async_bound", "dgpu_set_msa_async_bound")


def test_new_symbols_are_declared_and_exported():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "dgpu.h")).read(), flags=re.S)
    lib = delly_b200.lib()
    for s in NEW_SYMBOLS:
        assert re.search(r"\bint\s+" + s + r"\s*\(dgpu_ctx\*\s*ctx,\s*uint32_t\s+\w+,\s*uint32_t\s+\w+\)", txt), s
        assert hasattr(lib, s), s
    assert hasattr(delly_b200.Context, "set_ln_async_bound") and hasattr(delly_b200.Context, "set_msa_async_bound")


# ---------------------------------------------------------------------------------------------------------------------------------------
def _jobs_of(b):
    return [(b["seqs"][b["c_off"][i]:b["c_off"][i] + b["c_len"][i]].tobytes(), b["seqs"][b["r_off"][i]:b["r_off"][i] + b["r_len"][i]].tobytes())
            for i in range(len(b["c_off"]))]


def _sr_jobs(n=300, seed=21):
    return _jobs_of(synth.k3_consref_batch(n, seed=seed, cons_range=(150, 300), err=0.01, fast=True))   # about 225 x 900


def _lr_jobs(n=4, seed=22):
    return _jobs_of(synth.k3_consref_batch(n, seed=seed, cons_range=(2800, 3200), err=0.03, fast=True, ref_cap=10000))


def _iupac_jobs():
    jobs = [j for j in _jobs_of(_edge_batch(seed=7)) if len(j[0]) and len(j[1])]
    rng = np.random.default_rng(23)
    for c, r in _sr_jobs(20, seed=24):
        r = bytearray(r)
        r[int(rng.integers(0, len(r)))] = ord("R")
        jobs.append((c, bytes(r)))
    return jobs


def _wide_jobs(seed=25):
    rng = np.random.default_rng(seed)
    return [tuple(x.tobytes() for x in synth.wide_consref_job(rng, k, m, n))
            for k, m, n in (("del", 1500, 16900), ("dup", 3000, 24000), ("inv", 1200, 33000), ("del", 2500, 40000))]


class _Dev:
    """One longNeedle batch in device memory, with its output buffers."""

    def __init__(self, jobs, dev):
        import torch
        arena, off, ln = synth.pack([x for cr in jobs for x in cr])
        self.n = len(jobs)
        self.cap = (ln[0::2].astype(np.uint64) + ln[1::2].astype(np.uint64))
        aoff = np.concatenate([[0], np.cumsum(2 * self.cap)[:-1]]).astype(np.uint64)
        u32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint32).view(np.int32)).to(dev)   # noqa: E731
        self.seqs = torch.from_numpy(np.concatenate([arena, np.zeros(64, np.uint8)])).to(dev)
        self.c_off, self.c_len, self.r_off, self.r_len = u32(off[0::2]), u32(ln[0::2]), u32(off[1::2]), u32(ln[1::2])
        self.aln_off_np = aoff
        self.aln_off = torch.from_numpy(aoff.view(np.int64)).to(dev)
        self.aln = torch.zeros(int(2 * self.cap.sum()) + 64, dtype=torch.uint8, device=dev)
        self.aln_len = torch.zeros(self.n, dtype=torch.int32, device=dev)
        self.ok = torch.zeros(self.n, dtype=torch.uint8, device=dev)
        self.info = torch.zeros((self.n, 4), dtype=torch.int32, device=dev)

    def run(self, ctx, max_ref=None, stream=None):
        import torch
        self.aln.fill_(0x55); self.aln_len.fill_(-7); self.ok.fill_(7); self.info.fill_(-7)
        torch.cuda.synchronize()   # the fills run on torch's stream, the call on `stream` (None: the context's)
        ctx.long_needle_dev(self.seqs, self.c_off, self.c_len, self.r_off, self.r_len, self.aln, self.aln_off, self.aln_len, self.ok, self.info,
                            stream=stream, max_ref=max_ref)

    def result(self):
        """ok, aln_len, info and the alignment bytes (whole slots) of the last run."""
        import torch
        torch.cuda.synchronize()
        return (self.ok.cpu().numpy().copy(), self.aln_len.cpu().numpy().copy(), self.info.cpu().numpy().copy(), self.aln.cpu().numpy().copy())


def _same(x, y):
    return all(np.array_equal(a, b) for a, b in zip(x, y))


def _check_oracle(jobs, res, refused=()):
    ok, alen, info, aln = res
    O = po.oracle()
    off = np.concatenate([[0], np.cumsum([2 * (len(c) + len(r)) for c, r in jobs])[:-1]])
    for i, (c, r) in enumerate(jobs):
        if i in refused:
            assert ok[i] == 0 and alen[i] == 0 and info[i][2] == -1, i
            continue
        eok, e0, e1 = po.long_needle(O, c, r)
        assert info[i][2] != -1 and bool(ok[i]) == eok, (i, len(c), len(r))
        if eok:
            o, L, w = int(off[i]), int(alen[i]), len(c) + len(r)
            assert aln[o:o + L].tobytes() == e0 and aln[o + w:o + w + L].tobytes() == e1, (i, len(c), len(r))


@pytest.fixture
def fresh():
    """A context of its own (a bound holds workspace until its context closes)."""
    ctxs = []

    def make():
        ctxs.append(delly_b200.Context(0))
        return ctxs[-1]
    yield make
    for c in ctxs:
        c.close()


CASES = {"sr": (_sr_jobs, (400, 4000), None), "lr": (_lr_jobs, (4000, 12000), None), "iupac": (_iupac_jobs, (400, 4000), None),
         "wide": (_wide_jobs, (4000, 40000), 40000),
         "mixed": (lambda: _sr_jobs(60) + _lr_jobs(2) + _iupac_jobs() + _wide_jobs(), (4000, 40000), 40000)}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_bound_matches_synchronous_form_and_oracle(fresh, case):
    """dgpu_long_needle[_ex]_dev under the bound: ok, aln_len, info and every alignment byte equal the synchronous device form's, and the
    oracle's; the _ex form also for the shapes the plain form takes."""
    import torch
    make, bound, max_ref = CASES[case]
    jobs = make()
    d = _Dev(jobs, torch.device("cuda", 0))
    ctx = fresh()
    for mr in ([None, 40000] if max_ref is None else [max_ref]):
        d.run(ctx, max_ref=mr)
        want = d.result()
        ctx.set_ln_async_bound(*bound)
        d.run(ctx, max_ref=mr)
        got = d.result()
        ctx.set_ln_async_bound(0, 0)
        assert _same(got, want), (case, mr)
    _check_oracle(jobs, got)


@pytest.mark.gpu
@pytest.mark.parametrize("batch", ["long_needle", "long_needle_wide"])
def test_bound_on_the_existing_batches(fresh, batch):
    """The batches of test_long_needle.py (edge cases, the class bounds on both engines, the widest windows) and of test_long_needle_wide.py
    (DEL / DUP / INV windows of 16.4-40 kb), each in one call under a bound, against the synchronous form."""
    import torch
    rng = np.random.default_rng(77)
    if batch == "long_needle":
        jobs = [j for j in _jobs_of(_edge_batch()) if len(j[0]) and len(j[1])]
        for n in [b - 7 for k in range(1, 9) for b in (256 * k, 256 * k + 1)] + [b - 7 for k in range(4096, 16384, 2048) for b in (k, k + 1)] + [16377]:
            ref = synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]
            a = int(rng.integers(0, n // 3)); b = int(rng.integers(2 * n // 3, n - 60))
            cons = synth.sub_noise(rng, np.concatenate([ref[a:a + 60], ref[b:b + 60]]), 0.03)
            low = ref.copy(); low[n // 2] += 32
            jobs += [(cons.tobytes(), ref.tobytes()), (cons.tobytes(), low.tobytes())]
        bound, max_ref = (3000, 16377), None
    else:
        jobs = [tuple(x.tobytes() for x in synth.wide_consref_job(rng, k, m, n, noise=z))
                for k, m, n in (("del", 1000, 16378), ("del", 1500, 24000), ("del", 3000, 40000), ("dup", 4500, 18000), ("inv", 5000, 20000),
                                ("dup", 6000, 16900), ("del", 2500, 30000), ("inv", 1200, 33000)) for z in (0.02, 0.08)]
        bound, max_ref = (6000, 40000), 40000
    d = _Dev(jobs, torch.device("cuda", 0))
    ctx = fresh()
    d.run(ctx, max_ref=max_ref)
    want = d.result()
    ctx.set_ln_async_bound(*bound)
    d.run(ctx, max_ref=max_ref)
    assert _same(d.result(), want)


@pytest.mark.gpu
def test_calls_return_before_the_device_finishes(fresh):
    """Behind a long device sleep on the same stream, dgpu_msa_dev and dgpu_long_needle_ex_dev under their bounds return at once: the
    device is still sleeping when they are back (a call that synchronised would wait for the sleep)."""
    import torch
    dev = torch.device("cuda", 0)
    d = _Dev(_sr_jobs(200) + _wide_jobs()[:1], dev)
    m = _Msa(synth.k2_msa_batch(40, seed=31, fast=True), dev)
    ctx = fresh()
    ctx.set_ln_async_bound(400, 20000)
    ctx.set_msa_async_bound(32, 300)
    st = torch.cuda.Stream(device=dev)
    m.run(ctx, st.cuda_stream); d.run(ctx, max_ref=20000, stream=st.cuda_stream)   # warm-up: the per-job scratch
    torch.cuda.synchronize()
    want = d.result()
    d.aln_len.fill_(-7)
    torch.cuda.synchronize()
    ev = torch.cuda.Event()
    with torch.cuda.stream(st):
        torch.cuda._sleep(2_000_000_000)   # about a second
    t0 = time.perf_counter()
    m.run(ctx, st.cuda_stream)
    ctx.long_needle_dev(d.seqs, d.c_off, d.c_len, d.r_off, d.r_len, d.aln, d.aln_off, d.aln_len, d.ok, d.info, stream=st.cuda_stream, max_ref=20000)
    dt = time.perf_counter() - t0
    with torch.cuda.stream(st):
        ev.record()
    pending = not ev.query()
    torch.cuda.synchronize()
    assert pending and dt < 0.2, (pending, dt)
    assert _same(d.result(), want)


class _Msa:
    """One MSA batch in device memory, with its outputs (consensus at cons_base inside `buf`)."""

    def __init__(self, b, dev, buf=None, cons_base=0):
        import torch
        u32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint32).view(np.int32)).to(dev)   # noqa: E731
        self.b = b
        self.ncl = len(b["cluster_off"]) - 1
        rl = b["read_len"].astype(np.uint64)
        csum = np.concatenate([[0], np.cumsum(rl)])
        self.cap = (csum[b["cluster_off"][1:]] - csum[b["cluster_off"][:-1]]).astype(np.uint64)
        self.cons_off_np = np.concatenate([[0], np.cumsum(self.cap)[:-1]]).astype(np.uint64)
        self.seqs = torch.from_numpy(np.concatenate([b["seqs"], np.zeros(64, np.uint8)])).to(dev)
        self.read_off, self.read_len, self.cluster_off = u32(b["read_off"]), u32(b["read_len"]), u32(b["cluster_off"])
        self.cons_off = torch.from_numpy(self.cons_off_np.view(np.int64)).to(dev)
        self.buf = buf if buf is not None else torch.zeros(int(self.cap.sum()) + 64, dtype=torch.uint8, device=dev)
        self.cons_base = cons_base
        self.cons_len = torch.zeros(self.ncl, dtype=torch.int32, device=dev)
        self.n_rows = torch.zeros(self.ncl, dtype=torch.int32, device=dev)
        self.status = torch.zeros(self.ncl, dtype=torch.int32, device=dev)

    def run(self, ctx, stream=None):
        ctx.msa_dev(self.seqs, self.read_off, self.read_len, self.cluster_off, self.ncl, (5, -4, -10, -1), 2, self.buf.data_ptr() + self.cons_base,
                    self.cons_off, self.cons_len, self.n_rows, self.status, stream=stream)


def _chain(dev, seed):
    """MSA consensus of 24 clusters written into the longNeedle arena, each aligned against 3 windows of 500 - 20000 columns that contain
    part of its reads' haplotype (several wavefront classes and the wide class)."""
    import torch
    b = synth.k2_msa_batch(24, seed=seed, fast=True)
    rng = np.random.default_rng(seed)
    ncl = len(b["cluster_off"]) - 1
    widths = [500, 1500, 3000, 6000, 12000, 20000]
    wins = []
    for i in range(ncl):
        r0 = b["read_off"][b["cluster_off"][i]]
        read = b["seqs"][r0:r0 + b["read_len"][b["cluster_off"][i]]]
        for k in range(3):
            n = widths[(3 * i + k) % len(widths)]
            w = synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]
            p = int(rng.integers(0, n - len(read)))
            w[p:p + len(read)] = read
            wins.append(w)
    caps = b["read_len"].astype(np.uint64)
    cons_bytes = int(caps.sum()) + 64
    cons_base = 0
    ref_base = (cons_bytes + 255) & ~255
    ref_off = []
    o = ref_base
    for w in wins:
        ref_off.append(o); o += len(w)
    arena = torch.zeros(o + 64, dtype=torch.uint8, device=dev)
    arena[ref_base:o] = torch.from_numpy(np.concatenate(wins)).to(dev)
    m = _Msa(b, dev, buf=arena, cons_base=cons_base)
    cls = np.repeat(np.arange(ncl), 3)
    c_off = torch.from_numpy((m.cons_off_np[cls] + cons_base).astype(np.uint32).view(np.int32)).to(dev)
    r_len = np.array([len(w) for w in wins], np.uint32)
    cap = m.cap[cls] + r_len.astype(np.uint64)
    aln_off = np.concatenate([[0], np.cumsum(2 * cap)[:-1]]).astype(np.uint64)
    return dict(m=m, arena=arena, cls=torch.from_numpy(cls).to(dev), c_off=c_off, r_off=torch.from_numpy(np.array(ref_off, np.uint32).view(np.int32)).to(dev),
                r_len=torch.from_numpy(r_len.view(np.int32)).to(dev), aln_off=torch.from_numpy(aln_off.view(np.int64)).to(dev),
                aln=torch.zeros(int(2 * cap.sum()) + 64, dtype=torch.uint8, device=dev), c_len=torch.zeros(len(wins), dtype=torch.int32, device=dev),
                aln_len=torch.zeros(len(wins), dtype=torch.int32, device=dev), ok=torch.zeros(len(wins), dtype=torch.uint8, device=dev),
                info=torch.zeros((len(wins), 4), dtype=torch.int32, device=dev))


def _chain_run(ctx, c):
    """On torch's current stream, which must not be the default stream (a null stream means the context's stream to the library)."""
    import torch
    stream = torch.cuda.current_stream().cuda_stream
    assert stream
    c["m"].run(ctx, stream)
    torch.index_select(c["m"].cons_len, 0, c["cls"], out=c["c_len"])   # each window's consensus length, on the device
    ctx.long_needle_dev(c["arena"], c["c_off"], c["c_len"], c["r_off"], c["r_len"], c["aln"], c["aln_off"], c["aln_len"], c["ok"], c["info"],
                        stream=stream, max_ref=20000)


def _chain_result(c):
    import torch
    torch.cuda.synchronize()
    m = c["m"]
    return [t.cpu().numpy().copy() for t in (m.cons_len, m.n_rows, m.status, c["arena"], c["aln_len"], c["ok"], c["info"], c["aln"])]


def _chain_newdata(c, seed):
    """New reads (same lengths) and new window bases in the same buffers."""
    import torch
    rng = np.random.default_rng(seed)
    m = c["m"]
    s = m.b["seqs"].copy()
    s = synth.sub_noise(rng, s, 0.02)
    m.seqs[:len(s)] = torch.from_numpy(s).to(m.seqs.device)
    ref_base = int(c["r_off"][0].item())
    end = int(c["r_off"][-1].item()) + int(c["r_len"][-1].item())
    c["arena"][ref_base:end] = torch.from_numpy(synth._ACGT[rng.integers(0, 4, size=end - ref_base, dtype=np.uint8)]).to(c["arena"].device)


@pytest.mark.gpu
def test_msa_and_long_needle_capture_into_a_graph(fresh):
    """After one warm-up call, dgpu_msa_dev followed by dgpu_long_needle_ex_dev (consensus fed on the device into several wavefront classes
    and the wide class) is captured into a CUDA graph on the current stream; new data written into the same buffers and replayed gives the
    synchronous forms' results on that data. Two contexts on one device, each with its own graph."""
    import torch
    dev = torch.device("cuda", 0)
    ctxs = [fresh(), fresh()]
    chains = [_chain(dev, 41), _chain(dev, 42)]
    for ctx, c in zip(ctxs, chains):
        ctx.set_msa_async_bound(32, 300)
        ctx.set_ln_async_bound(400, 20000)
    graphs = []
    side = torch.cuda.Stream(device=dev)
    for ctx, c in zip(ctxs, chains):
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            _chain_run(ctx, c)   # warm-up: the per-job scratch
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            _chain_run(ctx, c)
        graphs.append(g)
    for k, c in enumerate(chains):
        _chain_newdata(c, 50 + k)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for g in graphs:
            g.replay()
    got = [_chain_result(c) for c in chains]
    ref = fresh()   # the synchronous forms, on the same buffers
    for c, r in zip(chains, got):
        with torch.cuda.stream(side):
            _chain_run(ref, c)
        want = _chain_result(c)
        assert (want[2] == 0).all()
        assert _same(r, want)


@pytest.mark.gpu
def test_refusals_under_the_bound(fresh):
    """Jobs beyond max_cons, beyond max_ref, beyond the call's max_ref and beyond the wavefront limits of the plain form each come back
    refused alone (ok = 0, aln_len = 0, info[2] = -1); every other job equals the synchronous form's, and dgpu_unsupported_count rises by
    exactly the number refused, once the work has finished."""
    import torch
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(61)
    sr = [j for j in _sr_jobs(60, seed=62) if len(j[0]) <= 300 and len(j[1]) <= 1200]
    for form, bound, max_ref in (("plain", (300, 1200), None), ("ex", (3000, 20000), 18000)):
        jobs = list(sr)
        bad = []

        def add(m, n):
            bad.append(len(jobs))
            ref = synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)]
            jobs.append((synth._ACGT[rng.integers(0, 4, size=m, dtype=np.uint8)].tobytes(), ref.tobytes()))
        if form == "plain":
            add(350, 800); add(200, 1300); add(301, 1201); add(3000, 17000)     # cons, ref, both beyond the bound; beyond the wavefront limits
        else:
            add(3500, 9000); add(2000, 21000); add(2000, 19000); add(1000, 16390)   # beyond max_cons, max_ref, the call's max_ref; inside
            bad.pop()
        d = _Dev(jobs, dev)
        ctx = fresh()
        d.run(ctx, max_ref=max_ref)
        want = d.result()
        ctx.set_ln_async_bound(*bound)
        n0 = ctx.unsupported
        d.run(ctx, max_ref=max_ref)
        got = d.result()
        assert ctx.unsupported == n0 + len(bad), form
        for i in range(len(jobs)):
            if i in bad:
                assert got[0][i] == 0 and got[1][i] == 0 and got[2][i][2] == -1, (form, i)
            else:
                assert got[0][i] == want[0][i] and got[1][i] == want[1][i] and np.array_equal(got[2][i], want[2][i]), (form, i)
        okmask = np.ones(len(jobs), bool); okmask[bad] = False
        for i in np.nonzero(okmask)[0]:
            o, L, w = int(d.aln_off_np[i]), int(got[1][i]), int(d.cap[i])
            assert np.array_equal(got[3][o:o + L], want[3][o:o + L]) and np.array_equal(got[3][o + w:o + w + L], want[3][o + w:o + w + L])


@pytest.mark.gpu
def test_switching_back_and_setter_arguments(fresh):
    """After (0, 0) the synchronous forms give the same results with the same launches as before the bound; out-of-range setter arguments
    and a plain-form call under a bound beyond its wavefront shapes return DGPU_ERR_ARG."""
    import torch
    ctx = fresh()
    lib = ctx._lib
    u = C.c_uint32
    for a, b in ((1, 65536), (16384, 100), (0, 100), (100, 0)):
        assert lib.dgpu_set_ln_async_bound(ctx.h, u(a), u(b)) == -2, (a, b)
    for a, b in ((1024, 100), (10, 1024), (0, 5), (5, 0)):
        assert lib.dgpu_set_msa_async_bound(ctx.h, u(a), u(b)) == -2, (a, b)
    d = _Dev(_sr_jobs(100, seed=71) + _lr_jobs(2, seed=72), torch.device("cuda", 0))
    m = _Msa(synth.k2_msa_batch(30, seed=73, fast=True), torch.device("cuda", 0))

    def both():
        l0 = ctx.launches
        m.run(ctx); d.run(ctx)
        r = d.result() + tuple(t.cpu().numpy() for t in (m.buf, m.cons_len, m.n_rows, m.status))
        return r, ctx.launches - l0
    want, lw = both()
    ctx.set_ln_async_bound(4000, 12000)
    ctx.set_msa_async_bound(64, 300)
    got, la = both()
    assert _same(got, want) and la > lw
    for bound in ((100, 20000), (16000, 16377)):
        ctx.set_ln_async_bound(*bound)
        with pytest.raises(delly_b200.DgpuError):
            d.run(ctx)
    ctx.set_ln_async_bound(0, 0)
    ctx.set_msa_async_bound(0, 0)
    again, l2 = both()
    assert _same(again, want) and l2 == lw
