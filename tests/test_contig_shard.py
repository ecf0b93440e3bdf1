"""`delly_b200 sr --shard-by contig`: every rank holds, scans, assembles and genotypes the alignments of its own contigs only, and the
per-contig logs (inter-chromosomal first observations, junction and pair logs, translocation split reads, decided junction-read jobs,
spanning events, read-depth) travel between the ranks (host/scan.hpp, host/assemble.hpp, host/genotype.hpp, host/gather.hpp).

The N-rank result must equal the single-process result record for record: every SV field, every genotype field, the GL bit patterns,
the consensus. dh_delly_sr_contig_sim hands each in-process rank ONLY the records of its own contigs, so equality also shows that no rank
needs an alignment it did not read. The sample is simulated here: three contigs with deletions, a tandem duplication, inversions and a
reciprocal translocation between contigs 1 and 2 (split reads with supplementary alignments on the other contig, inter-chromosomal pairs)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from test_host_genotype import _hash_string
from test_sharded import _contexts, _sites_from

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RL = 100
LIB = [100, 300, 15, 200, 400, 480]
CAP = 512
STRIDE = 1024


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _rc(a):
    return synth._revcomp(a)


def _simulate(seed=77, cov=24, pile=0):
    """Two haplotypes over contigs of 40, 30 and 30 kb. Haplotype A carries a deletion, a tandem duplication and an inversion on contig 0, an
    inversion on contig 1, a deletion on contig 2 and the reciprocal translocation chr1:15000 <-> chr2:12000; haplotype B the contig-0 deletion
    only (homozygous). 100 bp read pairs, insert ~ N(300, 15); a read over a piece boundary becomes a soft-clipped primary alignment of its
    longer part plus a hard-clipped supplementary alignment of the rest. pile: that many extra unpaired reads over the contig-2 deletion's
    left breakpoint (a contig with more junction-read jobs than one batch of the reference holds)."""
    rng = np.random.default_rng(seed)
    lens = [40000, 30000, 30000]
    ref = [synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)] for n in lens]
    hap_a = [[(0, 0, 8000, 1), (0, 9200, 21000, 1), (0, 20000, 32000, 1), (0, 32000, 33600, -1), (0, 33600, 40000, 1)],
             [(1, 0, 4000, 1), (1, 4000, 5300, -1), (1, 5300, 15000, 1), (2, 12000, 30000, 1)],
             [(2, 0, 5000, 1), (2, 5900, 12000, 1), (1, 15000, 30000, 1)]]
    hap_b = [[(0, 0, 8000, 1), (0, 9200, 40000, 1)], [(1, 0, 30000, 1)], [(2, 0, 30000, 1)]]
    recs, cigs, reads = [], [], []
    pid = 0

    def align(pieces, starts, a, strand):
        """(tid, pos, reverse, ops, ref-frame bases) of donor[a:a+RL] read on `strand`: primary first"""
        segs = []
        for (t, r0, r1, s), d0 in zip(pieces, starts):
            u, v = max(a, d0), min(a + RL, d0 + r1 - r0)
            if u < v:
                segs.append((t, r0, r1, s, d0, u, v))
        segs.sort(key=lambda g: -(g[6] - g[5]))
        out = []
        for k, (t, r0, r1, s, d0, u, v) in enumerate(segs[:2]):
            L, R = (u - a, a + RL - v) if s > 0 else (a + RL - v, u - a)
            pos = r0 + (u - d0) if s > 0 else r1 - (v - d0)
            out.append((t, pos, (strand * s) < 0, L, v - u, R, s))
        if len(out) == 2 and min(out[0][4], out[1][4]) < 20:
            out = out[:1]
        return out

    for hap in (hap_a, hap_b):
        for pieces in hap:
            donor = np.concatenate([ref[t][r0:r1] if s > 0 else _rc(ref[t][r0:r1]) for t, r0, r1, s in pieces])
            starts = np.cumsum([0] + [r1 - r0 for _, r0, r1, _ in pieces])[:-1]
            for _ in range(int(len(donor) * cov / (4 * RL))):
                ins = int(np.clip(rng.normal(300, 15), 220, 380))
                a1 = int(rng.integers(0, len(donor) - ins)); a2 = a1 + ins - RL
                al = [align(pieces, starts, a1, 1), align(pieces, starts, a2, -1)]
                seqs = [synth.sub_noise(rng, donor[x:x + RL].copy(), 0.003) for x in (a1, a2)]
                for k in (0, 1):
                    mt, mp, mrev = al[1 - k][0][0], al[1 - k][0][1], al[1 - k][0][2]
                    for ai, (t, pos, rev, L, M, R, s) in enumerate(al[k]):
                        bases = seqs[k] if s > 0 else _rc(seqs[k])
                        if ai == 0:
                            ops = ([(4, L)] if L else []) + [(0, M)] + ([(4, R)] if R else [])
                        else:
                            ops = ([(5, L)] if L else []) + [(0, M)] + ([(5, R)] if R else [])
                            bases = bases[L:L + M]
                        isize = 0 if t != mt else ((mp + RL - pos) if pos <= mp else -(pos + RL - mp))
                        flag = 0x1 | (0x40 if k == 0 else 0x80) | (0x10 if rev else 0) | (0x20 if mrev else 0) | (0x800 if ai else 0)
                        recs.append([t, pos, flag, 60, len(bases), len(cigs), len(ops), 0, mt, mp, isize, pid])
                        cigs.extend((ln << 4) | op for op, ln in ops)
                        reads.append(bases)
                pid += 1
    for i in range(pile):   # unpaired reference reads over chr2:5000
        pos = int(rng.integers(4920, 4960))
        recs.append([2, pos, 0, 60, RL, len(cigs), 1, 0, -1, -1, 0, pid + i])
        cigs.append((RL << 4) | 0)
        reads.append(ref[2][pos:pos + RL])
    off = np.cumsum([0] + [len(x) for x in reads])[:-1]
    r = np.array(recs, np.int64)
    r[:, 7] = off
    order = np.lexsort((np.arange(len(r)), r[:, 1], r[:, 0]))
    return dict(contig=np.concatenate(ref), coff=np.array([0, lens[0], lens[0] + lens[1]], np.uint32), clen=np.array(lens, np.uint32),
                rec=np.ascontiguousarray(r[order].astype(np.int32)), cig=np.array(cigs, np.uint32), reads=np.concatenate(reads).astype(np.uint8), npaired=pid)


def _keys(ref5, rec):
    ref5.ref_hash_sr_name.restype = C.c_uint64
    names = [f"q{int(r[11])}".encode() for r in rec]
    seeds = np.array([ref5.ref_hash_sr_name(nm, 1 if (int(r[2]) & 0x80) else 0) for nm, r in zip(names, rec)], np.uint64)
    nh = np.array([_hash_string(nm.decode()) if int(r[2]) & 0x1 else 0 for nm, r in zip(names, rec)], np.uint32)
    return seeds, nh


def _files(d, ref5, nfile):
    """the records dealt to nfile files by pair (file f: its records in coordinate order), with their read ids and name hashes"""
    rec = d["rec"]
    which = (rec[:, 11] % 5 < 2).astype(np.int64) if nfile == 2 else np.zeros(len(rec), np.int64)
    rec2 = np.ascontiguousarray(np.concatenate([rec[which == f] for f in range(nfile)]))
    off = np.array([0] + [int((which <= f).sum()) for f in range(nfile)], np.uint32)
    seeds, nh = _keys(ref5, rec2)
    return rec2, seeds, nh, off


def _run(H, handles, nranks, by_contig, d, files, geno=None, valid_intervals=None, site=None):
    rec, seeds, nh, off = files
    nfile = len(off) - 1
    lib = np.array([LIB] * nfile, np.int32)
    sv = np.zeros((CAP, 20), np.int32); fmt = np.zeros((nfile, CAP, 14), np.int32); gl = np.zeros((nfile, CAP, 3), np.float32)
    co = np.zeros((CAP, STRIDE), np.uint8); cl = np.zeros(CAP, np.int32)
    bounds = np.zeros(nranks + 1, np.uint64); held = np.zeros((nranks, 3), np.int64)
    g = geno if geno is not None else (None, None, None, None)
    s = site if site is not None else (None, None, None)
    arr = (C.c_void_p * nranks)(*[h if isinstance(h, int) else h.value for h in handles[:nranks]])
    n = H.dh_delly_sr_contig_sim(arr, nranks, by_contig, _p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 3, _p(rec), _p(seeds), _p(nh), _p(off), nfile,
                                 _p(g[0]), _p(g[1]), _p(g[2]), _p(g[3]), _p(d["cig"]), _p(d["reads"]), _p(lib), _p(valid_intervals), _p(s[0]),
                                 0 if site is None else len(s[0]), _p(s[1]), _p(s[2]), _p(sv), CAP, _p(fmt), _p(gl), _p(co), STRIDE, _p(cl), _p(bounds), _p(held))
    assert n != -100, "ranks disagree with each other"
    assert n > 0, n
    res = (n, sv[:n].copy(), fmt[:, :n].copy(), gl[:, :n].copy().view(np.uint32), [co[i, :cl[i]].tobytes() for i in range(n)])
    return res, bounds.astype(np.int64), held


def _same(a, b):
    assert a[0] == b[0]
    for k in (1, 2, 3):
        assert np.array_equal(a[k], b[k]), (k, np.argwhere(a[k] != b[k])[:5])
    assert a[4] == b[4]


def _check_held(bounds, held, total):
    """a rank was handed the records of its own contigs and nothing else; together the ranks hold every record once"""
    for r in range(len(held)):
        for t in range(held.shape[1]):
            if not (bounds[r] <= t < bounds[r + 1]):
                assert held[r, t] == 0, (r, t, held)
    assert held.sum() == total


@pytest.fixture(scope="module")
def sample():
    return _simulate()


@pytest.fixture(scope="module")
def keyed(sample, ref5):
    return {1: _files(sample, ref5, 1), 2: _files(sample, ref5, 2)}


@pytest.mark.parametrize("nranks", [2, 3, 5])
def test_contig_sharded_discovery_equals_single_process(hostdev, request, sample, keyed, nranks):
    """discovery + genotyping; N = 5 is more ranks than contigs (two ranks own none and still take part in every exchange)"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, nranks)
    one, _, _ = _run(H, handles, 1, 0, sample, keyed[1])
    got, bounds, held = _run(H, handles, nranks, 1, sample, keyed[1])
    _same(one, got)
    _check_held(bounds, held, len(sample["rec"]))
    svt = one[1][:, 15]
    assert {0, 1, 2, 3} <= set(svt.tolist()), svt                     # INV (both junction types), DEL, DUP
    tra = one[1][svt >= 5]
    assert len(tra) >= 2 and (tra[:, 0] != tra[:, 2]).all()           # inter-chromosomal calls
    assert (tra[:, 16] == 1).any()                                    # a translocation assembled from split reads of both contigs
    assert (one[1][:, 16] == 1).sum() >= 5
    if nranks == 5:
        assert (np.diff(bounds) == 0).sum() >= 2
    for m in keep:
        m.close()


@pytest.mark.parametrize("nranks", [2, 3, 5])
def test_contig_sharded_genotyping_mode_equals_single_process(hostdev, request, sample, keyed, nranks):
    """`delly sr -v sites.bcf`: the discovery calls as a shuffled site list, genotyped by contig"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, nranks)
    disc, _, _ = _run(H, handles, 1, 0, sample, keyed[1])
    site = _sites_from((disc[0], disc[1], None, None, disc[4]))
    one, _, _ = _run(H, handles, 1, 0, sample, keyed[1], site=site)
    got, bounds, held = _run(H, handles, nranks, 1, sample, keyed[1], site=site)
    _same(one, got)
    _check_held(bounds, held, len(sample["rec"]))
    for m in keep:
        m.close()


@pytest.mark.parametrize("nranks", [2, 3])
def test_contig_sharded_two_samples_equal_single_process(hostdev, request, sample, keyed, nranks):
    """two files in one call set: the scans pooled in file order, the genotyping per file"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, nranks)
    one, _, _ = _run(H, handles, 1, 0, sample, keyed[2])
    got, bounds, held = _run(H, handles, nranks, 1, sample, keyed[2])
    _same(one, got)
    _check_held(bounds, held, len(sample["rec"]))
    assert (one[2][1][:, 11] > 0).any()    # the second file has ALT junction reads of its own
    for m in keep:
        m.close()


@pytest.mark.parametrize("nranks", [2, 3])
def test_contig_sharded_exclude_set_equals_single_process(hostdev, request, sample, keyed, ref5, nranks):
    """an exclude set: contig 0 excluded as a whole (its mates are skipped by the scan) and chr2:20000-22000; scan, clustering and assembly
    see the valid regions, genotyping the whole contigs"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, nranks)
    rec, seeds, nh, off = keyed[1]
    valid = (rec[:, 0] != 0) & ~((rec[:, 0] == 2) & (rec[:, 1] >= 20000) & (rec[:, 1] < 22000))
    files = (np.ascontiguousarray(rec[valid]), seeds[valid].copy(), nh[valid].copy(), np.array([0, int(valid.sum())], np.uint32))
    valid_intervals = np.array([0, 1, 2], np.int32)   # the exclude set's valid regions per contig: none on contig 0
    one, _, _ = _run(H, handles, 1, 0, sample, files, geno=keyed[1], valid_intervals=valid_intervals)
    got, bounds, held = _run(H, handles, nranks, 1, sample, files, geno=keyed[1], valid_intervals=valid_intervals)
    _same(one, got)
    _check_held(bounds, held, int(valid.sum()) + len(rec))
    assert (one[1][:, 0] != 0).all() and one[0] >= 3
    for m in keep:
        m.close()


def test_contig_sharded_deep_contig_equals_single_process(hostdev, request, ref5):
    """more than 131072 junction-read jobs on one contig (the reference flushes its job buffer there): the decided jobs are merged in job order
    under the per-SV cap on every rank"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, 3)
    d = _simulate(pile=140000)
    files = _files(d, ref5, 1)
    one, _, _ = _run(H, handles, 1, 0, d, files)
    got, bounds, held = _run(H, handles, 3, 1, d, files)
    _same(one, got)
    _check_held(bounds, held, len(d["rec"]))
    hit = [i for i in range(one[0]) if one[1][i, 0] == 2 and one[1][i, 15] == 2 and one[1][i, 16] == 1 and abs(int(one[1][i, 1]) - 5000) < 20]
    assert hit, "the chr2 deletion under the pile is not a precise call"
    q = one[2][0][hit[0]]
    assert q[10] + q[11] == 250                  # junction reads capped at maxGenoReadCount
    for m in keep:
        m.close()


def test_contig_partition_is_contiguous_deterministic_and_balanced():
    H = delly_b200.hostlib()
    rng = np.random.default_rng(11)
    for n, r in ((24, 1), (24, 2), (24, 4), (24, 8), (3, 5), (1, 8), (84, 8), (25, 3)):
        w = rng.integers(1, 5_000_000, size=n).astype(np.uint64)
        if n > 3:
            w[0] *= 20   # one contig much larger than the rest
        b = np.zeros(r + 1, np.uint64)
        H.dh_partition_contigs(_p(w), n, r, _p(b))
        b2 = np.zeros(r + 1, np.uint64)
        H.dh_partition_contigs(_p(w), n, r, _p(b2))
        assert np.array_equal(b, b2)
        assert b[0] == 0 and b[-1] == n and (np.diff(b.astype(np.int64)) >= 0).all()
        parts = [int(w[int(b[i]):int(b[i + 1])].sum()) for i in range(r)]
        assert max(parts) <= int(w.sum()) / r + int(w.max())


def test_library_estimate_over_contig_shards_equals_single_process(sample):
    """getLibraryParams continued rank after rank from histograms, each rank holding its own contigs only"""
    H = delly_b200.hostlib()
    rec = sample["rec"]
    for nranks in (1, 2, 3, 5):
        a = np.zeros(7, np.int32); b = np.full(7, -7, np.int32)
        assert H.dh_library_params_contig_sim(nranks, _p(sample["clen"]), 3, _p(rec), len(rec), _p(a), _p(b)) == 0
        assert np.array_equal(a, b), (nranks, a, b)
        assert a[0] == RL and 280 <= a[1] <= 320


def test_library_estimate_stops_at_the_same_alignment_across_ranks():
    """a library characterized inside the second contig (1 M pairs screened): the screen stops on rank 1 and rank 2's contig, whose insert
    sizes differ, never enters the estimate"""
    H = delly_b200.hostlib()
    rng = np.random.default_rng(5)
    parts = []
    for tid, n, mu in ((0, 600_000, 300), (1, 500_000, 420), (2, 100_000, 900)):
        pos = np.sort(rng.integers(0, 5_000_000, size=n))
        isz = rng.normal(mu, 20, size=n).astype(np.int64)
        r = np.zeros((n, 12), np.int64)
        r[:, 0] = tid; r[:, 1] = pos; r[:, 2] = 0x1 | 0x40 | 0x20; r[:, 3] = 60; r[:, 4] = RL; r[:, 8] = tid; r[:, 9] = pos + isz - RL; r[:, 10] = isz
        parts.append(r)
    rec = np.ascontiguousarray(np.concatenate(parts).astype(np.int32))
    clen = np.array([5_100_000] * 3, np.uint32)
    for nranks in (1, 2, 3, 4):
        a = np.zeros(7, np.int32); b = np.full(7, -7, np.int32)
        assert H.dh_library_params_contig_sim(nranks, _p(clen), 3, _p(rec), len(rec), _p(a), _p(b)) == 0
        assert np.array_equal(a, b), (nranks, a, b)
    assert 310 <= a[1] <= 330   # index 500 k of the 600 k pairs at ~300 and the first 400 k at ~420


_WORKER = r'''
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, sys.argv[3]); sys.path.insert(0, os.path.join(sys.argv[3], "tests"))
import torch, torch.distributed as dist
rank, world = int(sys.argv[1]), int(sys.argv[2])
os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = sys.argv[4]
dist.init_process_group("gloo", rank=rank, world_size=world)
from delly_b200 import gather as dg
import test_contig_shard as T
z = np.load(sys.argv[6] + ".in.npz")
lib = C.CDLL(sys.argv[5])
lib.standin_ctx.restype = C.c_void_p
libc = C.CDLL(None); libc.malloc.restype = C.c_void_p; libc.malloc.argtypes = [C.c_size_t]
CB = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int))
def gather_cb(user, local, nbytes, all_p, counts_p, n_p):
    parts = dg.all_gather_bytes(C.string_at(local, nbytes) if nbytes else b"")
    blob = b"".join(parts)
    a = libc.malloc(max(len(blob), 1)); C.memmove(a, blob, len(blob))
    cnt = libc.malloc(8 * len(parts)); C.memmove(cnt, np.array([len(p) for p in parts], np.uint64).tobytes(), 8 * len(parts))
    all_p[0] = a; counts_p[0] = cnt; n_p[0] = len(parts)
    return 0
cb = CB(gather_cb)
p = T._p
CAP, ST = T.CAP, T.STRIDE
sv = np.zeros((CAP, 20), np.int32); fmt = np.zeros((1, CAP, 14), np.int32); gl = np.zeros((1, CAP, 3), np.float32)
co = np.zeros((CAP, ST), np.uint8); cl = np.zeros(CAP, np.int32); held = np.zeros(3, np.int64)
lib6 = np.array(T.LIB, np.int32)
n = lib.dh_delly_sr_contig_sharded(C.c_void_p(lib.standin_ctx()), p(z["contig"]), p(z["coff"]), p(z["clen"]), 3, p(z["rec"]), p(z["seeds"]), p(z["nh"]), p(z["off"]), 1,
                                   p(z["cig"]), p(z["reads"]), p(lib6), None, 0, None, None, rank, world, cb, None, p(sv), CAP, p(fmt), p(gl), p(co), ST, p(cl), p(held))
assert n > 0, n
np.savez(sys.argv[6] + ".%d.npz" % rank, n=n, sv=sv[:n], fmt=fmt[:, :n], gl=gl[:, :n], cl=cl[:n], co=co[:n], held=held)
dist.barrier(); dist.destroy_process_group()
'''


def test_world2_gloo_processes_contig_sharded_equal_single_process(standin, sample, keyed, tmp_path):
    """two real processes, each keeping the records of its own contigs; the exchange is torch.distributed (gloo) behind the gather callback"""
    ctxh = C.c_void_p(standin.standin_ctx())
    one, _, _ = _run(standin, [ctxh.value], 1, 0, sample, keyed[1])
    rec, seeds, nh, off = keyed[1]
    np.savez(str(tmp_path / "io") + ".in.npz", contig=sample["contig"], coff=sample["coff"], clen=sample["clen"], rec=rec, seeds=seeds, nh=nh, off=off,
             cig=sample["cig"], reads=sample["reads"])
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    so = os.path.join(HERE, "standin", "_build", "libhost_standin.so")
    port = str(27500 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), "2", ROOT, port, so, str(tmp_path / "io")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                              text=True) for r in range(2)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    held = []
    for r in range(2):
        z = np.load(str(tmp_path / "io") + ".%d.npz" % r)
        n = int(z["n"])
        _same(one, (n, z["sv"], z["fmt"], z["gl"].view(np.uint32), [z["co"][i, :z["cl"][i]].tobytes() for i in range(n)]))
        held.append(z["held"])
    held = np.array(held)
    assert held.sum() == len(rec) and ((held > 0).sum(axis=0) <= 1).all()   # every contig's records on one process only


# ---- the binding, one process: `delly_b200 sr --shard-by contig` takes the contig-sharded path (it exchanges with itself) ----------------
from test_bcf_parity import DELLY_REF, EX, _inflate, _run as _run_cmd, binding  # noqa: E402,F401  (binding: the [gpu] / [edlib-standin] fixture)


@pytest.mark.parametrize("mode", ["discovery", "genotyping"])
def test_binding_shard_by_contig_one_rank_bcf_identical_to_reference(binding, tmp_path, mode):
    """`delly_b200 sr --shard-by contig -g example/ref.fa example/sr.bam` (and -v sites.bcf) against the reference's own driver, byte for byte"""
    ref_out, our_out = str(tmp_path / "ref.bcf"), str(tmp_path / "ours.bcf")
    common = ["-g", os.path.join(EX, "ref.fa")]
    if mode == "genotyping":
        sites = str(tmp_path / "sites.bcf")
        _run_cmd([DELLY_REF, "sr"] + common + ["-o", sites, os.path.join(EX, "sr.bam")])
        common += ["-v", sites]
    _run_cmd([DELLY_REF, "sr"] + common + ["-o", ref_out, os.path.join(EX, "sr.bam")])
    r = _run_cmd([binding[0], "sr", "--shard-by", "contig"] + common + ["-o", our_out, os.path.join(EX, "sr.bam")])
    assert "rank 0/1: contigs 0-" in r.stderr
    a, b = _inflate(ref_out), _inflate(our_out)
    assert len(a) > 1000 and a == b, "BCF streams differ"
    assert open(ref_out + ".csi", "rb").read() == open(our_out + ".csi", "rb").read()


def test_binding_shard_by_refuses_dump_and_unknown_modes(binding, tmp_path):
    base = [binding[0], "sr", "-g", os.path.join(EX, "ref.fa"), "-o", str(tmp_path / "x.bcf")]
    for extra in (["--shard-by", "contig", "-d", str(tmp_path / "d.gz")], ["--shard-by", "reads"]):
        r = subprocess.run(base + extra + [os.path.join(EX, "sr.bam")], capture_output=True, text=True)
        assert r.returncode != 0 and "--shard-by" in r.stderr


def test_binding_read_share_only_splits_the_records(binding, tmp_path):
    """`--read-share-only`: every rank reads its own contigs and stops; the shares add up to the whole file, and nothing needs a device"""
    import json
    def share(n, r):
        t = str(tmp_path / ("t%d" % n))
        _run_cmd([binding[0], "sr", "--shard-by", "contig", "--nranks", str(n), "--rank", str(r), "--read-share-only", "--timing", t, "-g",
                  os.path.join(EX, "ref.fa"), os.path.join(EX, "sr.bam")])
        return json.load(open(t + ("." + str(r) if n > 1 else "")))
    whole = share(1, 0)["records"]
    parts = [share(3, r) for r in range(3)]
    assert whole > 1000 and sum(p["records"] for p in parts) == whole
    assert all(p["peak_rss_kb"] > 0 and "read_bam" in p["stages_ms"] for p in parts)
