"""`delly_b200 lr --shard-by contig`: every rank holds the long reads of its own contigs only. The junction logs, the read candidates of SVs
owned by higher ranks, the finished consensus records, the genotyping cap counts of SVs split over two ranks, the decided qualities,
read-depth and methylation sums, and the annotations travel between the ranks (host/pipeline.hpp, host/assemblelr.hpp, host/genotype.hpp,
host/gather.hpp).

The N-rank result must equal the single-process dellyLrCallMulti / dellyLrGenotype record for record: every SV field, consensus, alleles,
annotation, genotype field, GL bit pattern and methylation value. dh_delly_lr_contig_sim hands each in-process rank ONLY the records of its
own contigs, so equality also shows that no rank needs an alignment it did not read. The sample is simulated here: three contigs, deletions
and template insertions, a reciprocal translocation between contigs 1 and 2 whose split reads have their primary alignment on either contig
(more of them than a small -b and more than 4 x a small -p), and chimeric reads whose primary alignment on contig 0 carries a
deletion of contig 2 in a supplementary alignment."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from test_sharded import _contexts

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CAP = 256
STRIDE = 8192
ASTRIDE = 4096
# lr settings as tests/test_host_genotype.py::LR_CFG with -p 2 (maxCandidates 8) and -b 16 (the genotyping cap)
CFG = np.array([1, 25, 30, 75, 2, 1000, 2, 100, 10000, 400, 16, 25], np.int32)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _simulate(templates, seed=91, cov=18):
    """Haplotype A: a deletion and two template insertions on contig 0, a deletion on contig 2, the reciprocal translocation chr1:25000 <->
    chr2:20000; haplotype B: the contig-0 deletion and the translocation. Reads of 2-5 kb with 2 % substitutions; a read over a translocation junction is a
    soft-clipped primary alignment of its longer part plus a hard-clipped supplementary alignment of the rest; 18 more reads per translocation
    junction have their longer part, the primary alignment, on contig 1. Six chimeric reads join 1.5 kb of contig 0 (primary) to 1.2 kb over the
    contig-2 deletion (supplementary, the deletion in its CIGAR). Most reads carry an HP tag (their haplotype) and a PS tag (one of four phase
    sets). split[(junction, tid)]: the split reads of translocation junction 1 (chr1 -> chr2) or 2 (chr2 -> chr1) whose primary alignment is on
    contig tid."""
    rng = np.random.default_rng(seed)
    lens = [60000, 50000, 50000]
    ref = [synth._ACGT[rng.integers(0, 4, size=n, dtype=np.uint8)] for n in lens]
    ins1, ins2 = templates
    # a haplotype contig: pieces (tid, r0, r1) of the reference or (-1, sequence) insertions, all forward
    hap_a = [[(0, 0, 12000), (0, 12600, 30000), (-1, ins1), (0, 30000, 45000), (-1, ins2), (0, 45000, 60000)],
             [(1, 0, 25000), (2, 20000, 50000)],
             [(2, 0, 8000), (2, 8900, 20000), (1, 25000, 50000)]]
    hap_b = [[(0, 0, 12000), (0, 12600, 60000)], [(1, 0, 25000), (2, 20000, 50000)], [(2, 0, 20000), (1, 25000, 50000)]]
    recs, cigs, reads = [], [], []
    rid = [0]
    split = {}

    def emit(pieces, a, L, rev, hap, junction=None):
        """the alignments of donor[a:a+L] (primary first)"""
        segs, d0 = [], 0
        for pc in pieces:
            n = len(pc[1]) if pc[0] < 0 else pc[2] - pc[1]
            u, v = max(a, d0), min(a + L, d0 + n)
            if u < v:
                segs.append((pc, u - d0, v - d0, u - a))
            d0 += n
        # group consecutive pieces of one contig (with insertions between them) into one alignment
        groups = []
        for pc, s0, s1, q in segs:
            if groups and (pc[0] < 0 or groups[-1][0] == pc[0]):
                groups[-1][1].append((pc, s0, s1, q))
            elif pc[0] < 0:
                groups.append([None, [(pc, s0, s1, q)]])
            else:
                groups.append([pc[0], [(pc, s0, s1, q)]])
        groups = [g for g in groups if g[0] is not None]
        seq = np.concatenate([pc[1][s0:s1] if pc[0] < 0 else ref[pc[0]][pc[1] + s0:pc[1] + s1] for pc, s0, s1, q in segs])
        seq = synth.sub_noise(rng, seq, 0.02)
        out = []
        for tid, parts in groups:
            while parts and parts[-1][0][0] < 0:
                parts = parts[:-1]
            ops, pos, rp = [], None, None
            q0 = parts[0][3]
            for pc, s0, s1, q in parts:
                n = s1 - s0
                if pc[0] < 0:
                    ops.append((1, n))
                    continue
                r = pc[1] + s0
                if pos is None:
                    pos = r
                elif r > rp:
                    ops.append((2, r - rp))
                ops.append((0, n)); rp = r + n
            qe = parts[-1][3] + parts[-1][2] - parts[-1][1]
            out.append((tid, pos, ops, q0, qe, sum(n for o, n in ops if o == 0)))
        out.sort(key=lambda g: -g[5])
        if len(out) > 1 and out[1][5] < 300:
            out = out[:1]
        if junction is not None and len(out) == 2:
            split[(junction, out[0][0])] = split.get((junction, out[0][0]), 0) + 1
        hp = hap + 1 if rng.random() < 0.8 else 0
        ps = 100 + int(rng.integers(0, 4)) if hp else -1
        for k, (tid, pos, ops, q0, qe, _) in enumerate(out):
            clip = 5 if k else 4
            full = ([(clip, q0)] if q0 else []) + ops + ([(clip, L - qe)] if L - qe else [])
            bases = seq if k == 0 else seq[q0:qe]
            flag = (0x10 if rev else 0) | (0x800 if k else 0)
            recs.append([tid, pos, flag, 60, len(bases), len(cigs), len(full), 0, hp, ps, 0, rid[0]])
            cigs.extend((ln << 4) | op for op, ln in full)
            reads.append(bases)
        rid[0] += 1

    for h, hap in enumerate((hap_a, hap_b)):
        for k, pieces in enumerate(hap):
            n = sum(len(pc[1]) if pc[0] < 0 else pc[2] - pc[1] for pc in pieces)
            for _ in range(int(n * cov / (2 * 3500))):
                L = int(rng.integers(2000, 5001))
                emit(pieces, int(rng.integers(0, n - L)), L, bool(rng.integers(0, 2)), h, k if k else None)
            if k:   # junction reads with the longer part on contig 1 (the junction is where the last piece starts)
                at = n - (pieces[-1][2] - pieces[-1][1])
                for _ in range(9):
                    j = int(rng.integers(0, 200))
                    emit(pieces, at - 2400 - j if k == 1 else at - 1000 + j, 3400, bool(rng.integers(0, 2)), h, k)
    chim = [(0, 5000, 6500), (2, 7800, 8000), (2, 8900, 9900)]
    for _ in range(6):
        emit(chim, 0, 2700, bool(rng.integers(0, 2)), int(rng.integers(0, 2)))
    off = np.cumsum([0] + [len(x) for x in reads])[:-1]
    r = np.array(recs, np.int64)
    r[:, 7] = off
    order = np.lexsort((np.arange(len(r)), r[:, 1], r[:, 0]))
    return dict(contig=np.concatenate(ref), coff=np.array([0, lens[0], lens[0] + lens[1]], np.uint32), clen=np.array(lens, np.uint32),
                rec=np.ascontiguousarray(r[order].astype(np.int32)), cig=np.array(cigs, np.uint32), reads=np.concatenate(reads).astype(np.uint8),
                split=split)


@pytest.fixture(scope="module")
def tpl(ref8):
    from test_svanno import _templates
    seqs, arena, off = _templates(ref8)
    return seqs, arena, off


@pytest.fixture(scope="module")
def sample(tpl, ref9):
    from test_methyl import _with_tags
    alu, l1, sva, numt, ltr, hervk, polya = tpl[0]
    d = _with_tags(_simulate((np.concatenate([alu, polya[:25]]), ltr[:700])), 17)
    ref9.ref_hash_lr_name5.restype = C.c_uint64
    d["seeds"] = np.array([ref9.ref_hash_lr_name5(f"q{int(r[11])}".encode()) for r in d["rec"]], np.uint64)
    return d


def _files(d, nfile):
    """the records dealt to nfile files by read (a read's alignments stay in one file), with their tags"""
    rec = d["rec"]
    which = (rec[:, 11] % 3 == 0).astype(np.int64) if nfile == 2 else np.zeros(len(rec), np.int64)
    idx = np.concatenate([np.nonzero(which == f)[0] for f in range(nfile)])
    off = np.array([0] + [int((which <= f).sum()) for f in range(nfile)], np.uint32)
    mm_parts = [d["mm"][d["mm_off"][i]:d["mm_off"][i + 1]] for i in idx]
    ml_parts = [d["ml"][d["ml_off"][i]:d["ml_off"][i + 1]] for i in idx]
    return dict(rec=np.ascontiguousarray(rec[idx]), seeds=d["seeds"][idx].copy(), off=off, tagflags=d["tagflags"][idx].copy(),
                mm=np.concatenate(mm_parts + [np.zeros(1, np.uint8)]).astype(np.uint8), mm_off=np.cumsum([0] + [len(x) for x in mm_parts]).astype(np.uint32),
                ml=np.concatenate(ml_parts + [np.zeros(1, np.uint8)]).astype(np.uint8), ml_off=np.cumsum([0] + [len(x) for x in ml_parts]).astype(np.uint32))


def _run(H, handles, nranks, by_contig, d, f, tpl, valid=None, site=None, cfg=CFG):
    nfile = len(f["off"]) - 1
    sv = np.zeros((CAP, 20), np.int32); fmt = np.zeros((nfile, CAP, 14), np.int32); gl = np.zeros((nfile, CAP, 3), np.float32)
    co = np.zeros((CAP, STRIDE), np.uint8); cl = np.zeros(CAP, np.int32)
    an = np.zeros((CAP, 5), np.int32); me = np.zeros((nfile, CAP, 16), np.int32); al = np.zeros((CAP, ASTRIDE), np.uint8); all_ = np.zeros(CAP, np.int32)
    bounds = np.zeros(nranks + 1, np.uint64); held = np.zeros((nranks, 3), np.int64)
    s = site if site is not None else (None, None, None)
    arr = (C.c_void_p * nranks)(*[h if isinstance(h, int) else h.value for h in handles[:nranks]])
    n = H.dh_delly_lr_contig_sim(arr, nranks, by_contig, _p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 3, _p(f["rec"]), _p(f["seeds"]), _p(f["off"]), nfile,
                                 _p(valid), _p(d["cig"]), _p(d["reads"]), _p(cfg), C.c_float(0.9), C.c_float(0.5), _p(f["tagflags"]), _p(f["mm"]), _p(f["mm_off"]),
                                 _p(f["ml"]), _p(f["ml_off"]), 400, 128, 1, _p(tpl[1]), _p(tpl[2]), C.c_float(0.8), C.c_float(0.85), _p(s[0]),
                                 0 if site is None else len(s[0]), _p(s[1]), _p(s[2]), _p(sv), CAP, _p(fmt), _p(gl), _p(co), STRIDE, _p(cl), _p(an), _p(me),
                                 _p(al), ASTRIDE, _p(all_), _p(bounds), _p(held))
    assert n != -100, "ranks disagree with each other"
    assert n > 0, n
    res = (n, sv[:n].copy(), fmt[:, :n].copy(), gl[:, :n].copy().view(np.uint32), an[:n].copy(), me[:, :n].copy(),
           [co[i, :cl[i]].tobytes() for i in range(n)], [al[i, :all_[i]].tobytes() for i in range(n)])
    return res, bounds.astype(np.int64), held


def _same(a, b):
    assert a[0] == b[0]
    for k in (1, 2, 3, 4, 5):
        assert np.array_equal(a[k], b[k]), (k, np.argwhere(a[k] != b[k])[:5])
    assert a[6] == b[6] and a[7] == b[7]


def _check_held(bounds, held, total):
    for r in range(len(held)):
        for t in range(held.shape[1]):
            if not (bounds[r] <= t < bounds[r + 1]):
                assert held[r, t] == 0, (r, t, held)
    assert held.sum() == total


def _sites(one):
    """the discovery result as site rows (tests/test_genotype_mode.py), in shuffled file order"""
    from test_sharded import _sites_from
    return _sites_from((one[0], one[1], None, None, one[6]))


@pytest.mark.parametrize("nranks", [2, 3, 5])
def test_lr_contig_sharded_discovery_equals_single_process(hostdev, request, sample, tpl, nranks):
    """discovery + genotyping + annotation + methylation; N = 5 is more ranks than contigs (two ranks own none)"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, nranks)
    f = _files(sample, 1)
    one, _, _ = _run(H, handles, 1, 0, sample, f, tpl)
    got, bounds, held = _run(H, handles, nranks, 1, sample, f, tpl)
    _same(one, got)
    _check_held(bounds, held, len(sample["rec"]))
    sv, fmt = one[1], one[2][0]
    svt = sv[:, 15]
    assert {2, 4} <= set(svt.tolist()), svt
    tra = sv[svt >= 5]
    assert len(tra) >= 1 and (tra[:, 0] != tra[:, 2]).all() and (tra[:, 16] == 1).any()   # an assembled translocation
    # the read collection of a translocation ends on contig 2 (its owner's); on contig 1, walked before, each junction has more than twice
    # maxCandidates split reads with their primary alignment there, so the cap is reached before the owner's walk begins
    assert min(sample["split"].get((1, 1), 0), sample["split"].get((2, 1), 0)) > 2 * 4 * CFG[6], sample["split"]
    assert (tra[:, 0] == 2).all() and (tra[:, 2] == 1).all()
    assert (fmt[:, 8] % 100 > 0).any() and (fmt[:, 8] // 100 > 0).any() and (fmt[:, 9] >= 100).any()   # phased ALT reads, a phase set
    if nranks == 2:   # the -b cap binds: without it the translocations decide more reads
        free, _, _ = _run(H, handles, 1, 0, sample, f, tpl, cfg=np.where(np.arange(12) == 10, 250, CFG).astype(np.int32))
        assert free[0] == one[0]
        capped = fmt[:, 10] + fmt[:, 11]
        assert (capped[svt >= 5] <= CFG[10]).all() and (free[2][0][:, 10] + free[2][0][:, 11] > capped)[svt >= 5].any()
    assert (one[4][:, 1] > 0).any()                                                          # an insertion annotated from the templates
    assert (one[5] >= 0).any()                                                               # methylation calls
    assert any(sv[i, 0] == 2 and svt[i] == 2 and sv[i, 16] == 1 for i in range(one[0]))    # the contig-2 deletion, precise
    if nranks == 5:
        assert (np.diff(bounds) == 0).sum() >= 2
    for m in keep:
        m.close()


@pytest.mark.parametrize("nranks", [2, 3, 5])
def test_lr_contig_sharded_genotyping_mode_equals_single_process(hostdev, request, sample, tpl, nranks):
    """`delly lr -v sites.bcf`: the discovery calls as a shuffled site list (ids = file order), genotyped by contig"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, nranks)
    f = _files(sample, 1)
    disc, _, _ = _run(H, handles, 1, 0, sample, f, tpl)
    site = _sites(disc)
    one, _, _ = _run(H, handles, 1, 0, sample, f, tpl, site=site)
    got, bounds, held = _run(H, handles, nranks, 1, sample, f, tpl, site=site)
    _same(one, got)
    _check_held(bounds, held, len(sample["rec"]))
    for m in keep:
        m.close()


@pytest.mark.parametrize("nranks", [2, 3])
def test_lr_contig_sharded_two_samples_equal_single_process(hostdev, request, sample, tpl, nranks):
    """two files in one call set: discovery over the (contig, file, position) stream, genotyping and methylation per file"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, nranks)
    f = _files(sample, 2)
    one, _, _ = _run(H, handles, 1, 0, sample, f, tpl)
    got, bounds, held = _run(H, handles, nranks, 1, sample, f, tpl)
    _same(one, got)
    _check_held(bounds, held, len(sample["rec"]))
    assert (one[2][1][:, 11] > 0).any()
    for m in keep:
        m.close()


@pytest.mark.parametrize("nranks", [2, 3])
def test_lr_contig_sharded_exclude_set_equals_single_process(hostdev, request, sample, tpl, nranks):
    """an exclude set (chr0:40000-50000): discovery sees the valid regions, genotyping the whole contigs"""
    H, ctxh = hostdev
    handles, keep = _contexts(request.node.callspec.params["hostdev"], H, ctxh, nranks)
    f = _files(sample, 1)
    rec = f["rec"]
    valid = (~((rec[:, 0] == 0) & (rec[:, 1] >= 40000) & (rec[:, 1] < 50000))).astype(np.uint8)
    one, _, _ = _run(H, handles, 1, 0, sample, f, tpl, valid=valid)
    got, bounds, held = _run(H, handles, nranks, 1, sample, f, tpl, valid=valid)
    _same(one, got)
    _check_held(bounds, held, int(valid.sum()) + len(rec))
    for m in keep:
        m.close()


_WORKER = r'''
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, sys.argv[3]); sys.path.insert(0, os.path.join(sys.argv[3], "tests"))
import torch, torch.distributed as dist
rank, world = int(sys.argv[1]), int(sys.argv[2])
os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = sys.argv[4]
dist.init_process_group("gloo", rank=rank, world_size=world)
from delly_b200 import gather as dg
import test_lr_contig_shard as T
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
CAP = T.CAP
sv = np.zeros((CAP, 20), np.int32); fmt = np.zeros((1, CAP, 14), np.int32); gl = np.zeros((1, CAP, 3), np.float32)
co = np.zeros((CAP, T.STRIDE), np.uint8); cl = np.zeros(CAP, np.int32); held = np.zeros(3, np.int64)
an = np.zeros((CAP, 5), np.int32); me = np.zeros((1, CAP, 16), np.int32); al = np.zeros((CAP, T.ASTRIDE), np.uint8); all_ = np.zeros(CAP, np.int32)
n = lib.dh_delly_lr_contig_sharded(C.c_void_p(lib.standin_ctx()), p(z["contig"]), p(z["coff"]), p(z["clen"]), 3, p(z["rec"]), p(z["seeds"]), p(z["off"]), 1,
                                   p(z["cig"]), p(z["reads"]), p(T.CFG), C.c_float(0.9), C.c_float(0.5), p(z["tagflags"]), p(z["mm"]), p(z["mm_off"]), p(z["ml"]),
                                   p(z["ml_off"]), 400, 128, 1, p(z["tpl_arena"]), p(z["tpl_off"]), C.c_float(0.8), C.c_float(0.85), rank, world, cb, None,
                                   p(sv), CAP, p(fmt), p(gl), p(co), T.STRIDE, p(cl), p(an), p(me), p(al), T.ASTRIDE, p(all_), p(held))
assert n > 0, n
np.savez(sys.argv[6] + ".%d.npz" % rank, n=n, sv=sv[:n], fmt=fmt[:, :n], gl=gl[:, :n], an=an[:n], me=me[:, :n], cl=cl[:n], co=co[:n], al=al[:n], all_=all_[:n], held=held)
dist.barrier(); dist.destroy_process_group()
'''


def test_world2_gloo_processes_lr_contig_sharded_equal_single_process(standin, sample, tpl, tmp_path):
    """two real processes, each keeping the long reads of its own contigs; the exchange is torch.distributed (gloo) behind the gather callback"""
    ctxh = C.c_void_p(standin.standin_ctx())
    f = _files(sample, 1)
    one, _, _ = _run(standin, [ctxh.value], 1, 0, sample, f, tpl)
    np.savez(str(tmp_path / "io") + ".in.npz", contig=sample["contig"], coff=sample["coff"], clen=sample["clen"], cig=sample["cig"], reads=sample["reads"],
             tpl_arena=tpl[1], tpl_off=tpl[2], **f)
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    so = os.path.join(HERE, "standin", "_build", "libhost_standin.so")
    port = str(29600 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), str(r), "2", ROOT, port, so, str(tmp_path / "io")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                              text=True) for r in range(2)]
    outs = [p.communicate(timeout=900)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    held = []
    for r in range(2):
        z = np.load(str(tmp_path / "io") + ".%d.npz" % r)
        n = int(z["n"])
        _same(one, (n, z["sv"], z["fmt"], z["gl"].view(np.uint32), z["an"], z["me"], [z["co"][i, :z["cl"][i]].tobytes() for i in range(n)],
                    [z["al"][i, :z["all_"][i]].tobytes() for i in range(n)]))
        held.append(z["held"])
    held = np.array(held)
    assert held.sum() == len(f["rec"]) and ((held > 0).sum(axis=0) <= 1).all()


# ---- the binding, one process: `delly_b200 lr --shard-by contig` takes the contig-sharded path (it exchanges with itself) ----------------
from test_bcf_parity import DELLY_REF, EX, _inflate, _run as _run_cmd, binding  # noqa: E402,F401  (binding: the [gpu] / [edlib-standin] fixture)


@pytest.mark.parametrize("mode", ["discovery", "genotyping"])
def test_binding_lr_shard_by_contig_one_rank_bcf_identical_to_reference(binding, tmp_path, mode):
    """`delly_b200 lr --shard-by contig -g example/ref.fa example/lr.bam` (and -v sites.bcf) against the reference's own driver, byte for byte"""
    ref_out, our_out = str(tmp_path / "ref.bcf"), str(tmp_path / "ours.bcf")
    common = ["-g", os.path.join(EX, "ref.fa")]
    if mode == "genotyping":
        sites = str(tmp_path / "sites.bcf")
        _run_cmd([DELLY_REF, "lr"] + common + ["-o", sites, os.path.join(EX, "lr.bam")])
        common += ["-v", sites]
    _run_cmd([DELLY_REF, "lr"] + common + ["-o", ref_out, os.path.join(EX, "lr.bam")])
    r = _run_cmd([binding[0], "lr", "--shard-by", "contig"] + binding[1:] + common + ["-o", our_out, os.path.join(EX, "lr.bam")])
    assert "rank 0/1: contigs 0-" in r.stderr
    a, b = _inflate(ref_out), _inflate(our_out)
    assert len(a) > 1000 and a == b, "BCF streams differ"
    assert open(ref_out + ".csi", "rb").read() == open(our_out + ".csi", "rb").read()


def test_binding_lr_shard_by_contig_refuses_dump(binding, tmp_path):
    r = subprocess.run([binding[0], "lr", "--shard-by", "contig", "-d", str(tmp_path / "d.gz"), "-g", os.path.join(EX, "ref.fa"), "-o", str(tmp_path / "x.bcf"),
                        os.path.join(EX, "lr.bam")], capture_output=True, text=True)
    assert r.returncode != 0 and "--shard-by" in r.stderr


SIMBAM = os.path.join(ROOT, "delly_b200", "bin", "simbam")


@pytest.fixture(scope="module")
def lrsim(tmp_path_factory):
    """a three-contig long-read sample (3 kb reads) from tools/simbam.cpp"""
    pre = str(tmp_path_factory.mktemp("lrsim") / "lrs")
    _run_cmd([SIMBAM, "--out", pre, "--genome-len", "600000", "--contigs", "3", "--n-sv", "30", "--cov", "12", "--read-len", "3000", "--isize", "8000",
              "--isd", "300", "--err", "0.01", "--seed", "7", "--types", "DEL,DUP,INV", "--threads", "4"])
    return pre


@pytest.mark.parametrize("mode", ["discovery", "genotyping"])
def test_binding_lr_shard_by_contig_three_contigs_bcf_identical_to_reference(binding, tmp_path, lrsim, mode):
    """`delly_b200 lr --shard-by contig` on a three-contig sample (and -v sites.bcf) against the reference's own driver, byte for byte"""
    ref_out, our_out = str(tmp_path / "ref.bcf"), str(tmp_path / "ours.bcf")
    common = ["-g", lrsim + ".fa"]
    if mode == "genotyping":
        sites = str(tmp_path / "sites.bcf")
        _run_cmd([DELLY_REF, "lr"] + common + ["-o", sites, lrsim + ".bam"])
        common += ["-v", sites]
    _run_cmd([DELLY_REF, "lr"] + common + ["-o", ref_out, lrsim + ".bam"])
    r = _run_cmd([binding[0], "lr", "--shard-by", "contig"] + binding[1:] + common + ["-o", our_out, lrsim + ".bam"])
    assert "rank 0/1: contigs 0-2" in r.stderr
    a, b = _inflate(ref_out), _inflate(our_out)
    assert len(a) > 1000 and a == b, "BCF streams differ"
    assert sum(a.count(k) for k in (b"DEL0", b"DUP0", b"INV0")) >= 10   # the record IDs
    assert open(ref_out + ".csi", "rb").read() == open(our_out + ".csi", "rb").read()


def test_binding_lr_read_share_only_splits_the_records(binding, tmp_path, lrsim):
    """`lr --read-share-only` on three contigs: every rank reads its own contigs and stops, and nothing needs a device. The records of one
    contig are measured as the share of a rank owning that contig alone (three ranks: one contig each); every rank of a two-rank cut then holds
    exactly the records of the contigs its stderr line names, and the shares add up to the whole file."""
    import json
    import re

    def share(n, r):
        t = str(tmp_path / ("t%d" % n))
        p = _run_cmd([binding[0], "lr", "--shard-by", "contig", "--nranks", str(n), "--rank", str(r), "--read-share-only", "--timing", t] + binding[1:] +
                     ["-g", lrsim + ".fa", lrsim + ".bam"])
        m = re.search(r"rank %d/%d: contigs (\d+)-(\d+) .*, (\d+) records" % (r, n), p.stderr)
        assert m, p.stderr
        j = json.load(open(t + ("." + str(r) if n > 1 else "")))
        assert j["records"] == int(m.group(3)) and j["peak_rss_kb"] > 0 and "read_bam" in j["stages_ms"]
        return int(m.group(1)), int(m.group(2)), j["records"]
    whole = share(1, 0)
    assert whole[:2] == (0, 2) and whole[2] > 1000
    per_contig = {}
    for r in range(3):
        lo, hi, n = share(3, r)
        assert lo == hi == r, (r, lo, hi)
        per_contig[r] = n
    assert all(v > 0 for v in per_contig.values()) and sum(per_contig.values()) == whole[2]
    two = [share(2, r) for r in range(2)]
    assert two[0][0] == 0 and two[0][1] + 1 == two[1][0] and two[1][1] == 2
    for lo, hi, n in two:
        assert n == sum(per_contig[t] for t in range(lo, hi + 1))
