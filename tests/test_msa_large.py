"""msa (src/msa.h:185-239) on clusters of more than 32 reads: the oracle against the compiled reference (CPU), msa_large_kernel against the
oracle (GPU), and the two consumers of large clusters end to end: the split-read assembly stage (translocation clusters are not capped
by maxReadPerSV, src/shortpe.h:140) and `delly sr -p 200` on a deep sample."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import delly_b200
from delly_b200 import synth
from oracle import pyoracle as po
from test_bcf_parity import DELLY_REF, EX, HERE, REFDIR, ROOT, _inflate, _run
from test_host_split import _genome, _p, _sv_cases

STANDIN = os.path.join(HERE, "standin")


def _build_standin(out_name, sources, shared):
    """the CPU suite's stand-in of the C ABI (tests/standin) with dgpu_msa_ex served as well (msa_ex_standin.cpp), built next to the tests"""
    out = os.path.join(STANDIN, "_build")
    os.makedirs(out, exist_ok=True)
    target = os.path.join(out, out_name)
    pkg = os.path.join(ROOT, "delly_b200")
    srcs = [os.path.join(STANDIN, s) for s in sources] + [os.path.join(STANDIN, "msa_ex_standin.cpp")]
    deps = srcs + [os.path.join(STANDIN, "host_standin.cpp")] + [os.path.join(pkg, "host", f) for f in os.listdir(os.path.join(pkg, "host"))]
    deps += [os.path.join(ROOT, "bindings", f) for f in os.listdir(os.path.join(ROOT, "bindings"))]
    if not os.path.exists(target) or os.path.getmtime(target) < max(os.path.getmtime(f) for f in deps):
        delly_b200.lib()   # every other entry point links against the CUDA library
        cmd = ["g++", "-std=c++17", "-O2", "-w"] + (["-fPIC", "-shared", "-Wl,-Bsymbolic"] if shared else []) + ["-o", target] + srcs
        cmd += ["-L" + REFDIR, "-l:libdelly_ref.so", "-L" + pkg, "-l:libdelly_b200.so", "-Wl,-rpath," + REFDIR, "-Wl,-rpath," + pkg]
        if not shared:
            hts = os.path.join(REFDIR, "hts")
            cmd = cmd[:4] + ["-I" + os.path.join(hts, "include")] + cmd[4:] + [os.path.join(hts, "libhts.a"), "-lz", "-lm", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return target


@pytest.fixture(params=[pytest.param("gpu", marks=pytest.mark.gpu), "edlib-standin"])
def hostdev_large(request, ref):
    """(host library, context handle): the real libraries on an H100, or the CPU stand-in with dgpu_msa_ex forwarded to the reference's msa"""
    if request.param == "gpu":
        return delly_b200.hostlib(), request.getfixturevalue("ctx").h
    lib = C.CDLL(_build_standin("libhost_standin_msa_ex.so", ["host_standin.cpp"], shared=True))
    lib.standin_ctx.restype = C.c_void_p
    return lib, C.c_void_p(lib.standin_ctx())


@pytest.fixture(params=[pytest.param("gpu", marks=pytest.mark.gpu), "edlib-standin"])
def binding_large(request):
    """the drop-in program: the real binary on an H100, or the binding compiled over the CPU stand-in with dgpu_msa_ex served"""
    assert os.path.exists(DELLY_REF) and os.path.isdir(EX), "oracle/_ref/delly_ref missing: run __graft_entry__.build() where /root/reference exists"
    if request.param == "gpu":
        exe = os.path.join(ROOT, "delly_b200", "bin", "delly_b200")
        assert os.path.exists(exe), "delly_b200/bin/delly_b200 not built"
        return exe
    po.build()
    return _build_standin("delly_b200_standin_msa_ex", ["binding_standin.cpp"], shared=False)


def _batch(clusters):
    reads, coff = [], [0]
    for c in clusters:
        reads += c
        coff.append(len(reads))
    arena, off, ln = synth.pack(reads)
    return dict(seqs=arena, read_off=off, read_len=ln, cluster_off=np.array(coff, np.uint32))


def _clusters(b):
    for i in range(len(b["cluster_off"]) - 1):
        yield [b["seqs"][b["read_off"][r]: b["read_off"][r] + b["read_len"][r]].tobytes()
               for r in range(b["cluster_off"][i], b["cluster_off"][i + 1])]


def _tiling(rng, n, lo, hi, span, err=0.01, n_rate=0.0):
    """n reads of lo..hi bp at random offsets of one random haplotype of span bp, with substitutions and optional N bases"""
    hap = synth._ACGT[rng.integers(0, 4, size=span)]
    out = []
    for _ in range(n):
        L = int(rng.integers(lo, hi + 1))
        s = int(rng.integers(0, span - L + 1))
        r = hap[s:s + L].copy()
        sub = rng.random(L) < err
        r[sub] = synth._ACGT[rng.integers(0, 4, size=int(sub.sum()))]
        r[rng.random(L) < n_rate] = ord("N")
        out.append(r.tobytes())
    return out


def _large_clusters():
    """33 .. 300 read clusters: identical reads, N bases, reads > 256 bp (plain-DP LCS), alignments wider than one 256-column strip,
    many distinct column profiles"""
    rng = np.random.default_rng(61)
    same = _tiling(rng, 1, 120, 120, 120)[0]
    return [
        [same] * 40,
        _tiling(rng, 33, 100, 150, 260),
        _tiling(rng, 40, 280, 300, 420, err=0.005),             # every pair longer than the bit-parallel LCS width
        _tiling(rng, 64, 140, 150, 400, n_rate=0.01),
        _tiling(rng, 100, 150, 150, 390, err=0.02),
        _tiling(rng, 200, 100, 150, 300),
        _tiling(rng, 300, 150, 150, 380, err=0.005),
    ]


def _check(ctx, b, mc=2, max_reads=delly_b200.MSA_LARGE_MAXR):
    cons, nrows, status, alns = ctx.msa(b["seqs"], b["read_off"], b["read_len"], b["cluster_off"], min_clique=mc, want_alignment=True,
                                        max_reads=max_reads)
    O = po.oracle()
    for i, reads in enumerate(_clusters(b)):
        rows, ecs, ealn = po.msa(O, reads, mc, want_alignment=True)
        assert alns[i] == ealn, (i, len(reads))
        assert cons[i] == ecs, (i, len(reads))
        assert nrows[i] == rows


def test_oracle_matches_reference_large_clusters(ref):
    """the oracle is a valid checker at these sizes: the reference's msa compiled verbatim gives the same alignments and consensus"""
    O = po.oracle()
    cl = _large_clusters()
    for reads in cl[:5] + [cl[5][:120]]:
        for mc in (2, 3):
            assert po.msa(O, reads, mc, want_alignment=True) == po.msa(ref, reads, mc, want_alignment=True), (len(reads), mc)


@pytest.mark.gpu
def test_cuda_large_clusters_match_oracle(ctx):
    _check(ctx, _batch(_large_clusters()))
    _check(ctx, _batch(_large_clusters()[:3]), mc=3)


@pytest.mark.gpu
def test_cuda_mixed_batch_runs_both_kernels(ctx):
    """small clusters (one warp each) and large ones (one CTA each) in one call, interleaved"""
    small = list(_clusters(synth.k2_msa_batch(24, seed=62, read_len=150, max_off=120, err=0.01)))
    rng = np.random.default_rng(63)
    large = [_tiling(rng, int(rng.integers(33, 90)), 120, 150, 330) for _ in range(6)]
    mixed = []
    for i, c in enumerate(small):
        mixed.append(c)
        if i % 4 == 1:
            mixed.append(large[i // 4])
    _check(ctx, _batch(mixed))


@pytest.mark.gpu
def test_cuda_cluster_at_read_cap(ctx):
    """1023 reads (the cap) equal the oracle; 1024 reads, or more than max_reads, get status 1 alone; max_reads 0 or 1024 is refused"""
    rng = np.random.default_rng(64)
    cap = _tiling(rng, 1023, 50, 70, 110, err=0.01)
    _check(ctx, _batch([cap]))

    mid = _tiling(rng, 40, 100, 150, 250)
    over = _tiling(rng, 1024, 50, 70, 110)
    b = _batch([mid, over, mid[:10], _tiling(rng, 150, 60, 80, 140)])
    cons, nrows, status = ctx.msa(b["seqs"], b["read_off"], b["read_len"], b["cluster_off"], check=False, max_reads=delly_b200.MSA_LARGE_MAXR)
    assert status.tolist() == [0, 1, 0, 0] and cons[1] == b"" and nrows[1] == 0
    cons2, nrows2, status2 = ctx.msa(b["seqs"], b["read_off"], b["read_len"], b["cluster_off"], check=False, max_reads=100)
    assert status2.tolist() == [0, 1, 0, 1] and cons2[3] == b"" and nrows2[3] == 0
    O = po.oracle()
    for i, reads in ((0, mid), (2, mid[:10])):
        rows, ecs, _ = po.msa(O, reads, 2)
        assert cons[i] == ecs == cons2[i] and nrows[i] == rows == nrows2[i]

    lib = ctx._lib
    n = len(b["cluster_off"]) - 1
    cl = np.zeros(n, np.uint32); nr = np.zeros(n, np.uint32); st = np.zeros(n, np.uint32)
    cap_bytes = int(b["read_len"].sum())
    out = np.zeros(cap_bytes, np.uint8)
    co = np.concatenate([[0], np.cumsum([sum(len(r) for r in c) for c in _clusters(b)])[:-1]]).astype(np.uint64)
    for bad in (0, 1024):
        rc = lib.dgpu_msa_ex(ctx.h, _p(b["seqs"]), C.c_uint64(b["seqs"].nbytes), _p(b["read_off"]), _p(b["read_len"]), C.c_uint32(len(b["read_off"])),
                             _p(b["cluster_off"]), C.c_uint32(n), 5, -4, -10, -1, 2, _p(out), _p(co), C.c_uint64(cap_bytes), _p(cl), _p(nr), _p(st),
                             None, None, C.c_uint64(0), None, C.c_uint32(bad))
        assert rc == -2 and b"max_reads" in lib.dgpu_last_error(ctx.h)


# ---- split-read assembly stage with large clusters ------------------------------------------------------------------------

def _large_assembly_case(seed, big_tra, nsv=24):
    """_assembly_case of test_host_split with 40 .. 150 distinct split reads on the translocations (big_tra) or on every other SV type"""
    rng = np.random.default_rng(seed)
    g1, g2 = _genome(seed + 1), _genome(seed + 2)
    svs, cons = _sv_cases(seed + 3, g1, g2, n=nsv, cons_range=(220, 330), with_ins=True)
    recs, cigs, reads, store = [], [], [], []
    name = [0]

    def add(tid, pos, seq, svid):
        f = (0x80 if rng.random() < 0.5 else 0x40) | 0x1
        recs.append([tid, pos, f, 60, len(seq), len(cigs), 1, sum(len(r) for r in reads), tid, pos + 200, 0, name[0]])
        cigs.append((len(seq) << 4) | 0)
        reads.append(seq)
        store.append([tid, pos, name[0], 1 if (f & 0x80) else 0, svid])
        name[0] += 1

    for i in range(len(svs)):
        chr_, s, chr2, e, svt, ins = [int(x) for x in svs[i]]
        c = cons[i] if rng.random() < 0.5 else synth.revcomp(cons[i])
        k = int(rng.integers(40, 151)) if (svt >= 5) == big_tra else int(rng.choice([0, 1, 5, 12]))
        for _ in range(k):
            rl = int(rng.integers(100, 151)); st = int(rng.integers(0, len(c) - rl + 1))
            w = synth.sub_noise(rng, c[st:st + rl].copy(), 0.01)
            second = rng.random() < 0.3
            if svt == 0 and second: tid, pos, seq = chr_, s + int(rng.integers(0, 40)), synth.revcomp(w)
            elif svt == 1 and second: tid, pos, seq = chr_, e + int(rng.integers(0, 40)), synth.revcomp(w)
            elif svt == 5: tid, pos, seq = (chr2, e - 60, synth.revcomp(w)) if second else (chr_, s - 60, w)
            elif svt == 6: tid, pos, seq = (chr2, e - 60, w) if second else (chr_, s - 60, synth.revcomp(w))
            elif svt >= 7: tid, pos, seq = (chr2, e - 60, w) if second else (chr_, s - 60, w)
            else: tid, pos, seq = chr_, max(s - 100, 0), w
            add(tid, pos, seq, i)
    rec = np.array(recs, np.int64)
    order = np.lexsort((np.arange(len(rec)), rec[:, 1], rec[:, 0]))
    rec = np.ascontiguousarray(rec[order].astype(np.int32))
    contig = np.frombuffer(g1 + g2, np.uint8).copy()
    sv7 = np.array([[svs[i][0], svs[i][1], svs[i][2], svs[i][3], svs[i][4], svs[i][5], i] for i in range(len(svs))], np.int32)
    return dict(contig=contig, coff=np.array([0, len(g1)], np.uint32), clen=np.array([len(g1), len(g2)], np.uint32), rec=rec, cig=np.array(cigs, np.uint32),
                reads=np.concatenate(reads).astype(np.uint8), store=np.array(store, np.int32), sv=sv7)


@pytest.mark.parametrize("big_tra,max_per_sv", [(True, 20), (False, 100)])
def test_assemble_split_reads_large_clusters_match_reference(hostdev_large, ref5, big_tra, max_per_sv):
    """translocations with 40 .. 150 split reads at maxReadPerSV = 20 (their store is uncapped), other SVs at maxReadPerSV = 100:
    every output field equals assembleSplitReads run verbatim"""
    H, ctxh = hostdev_large
    d = _large_assembly_case(7100 + int(big_tra), big_tra)
    n, nrec = len(d["sv"]), len(d["rec"])
    outs = []
    for fn, lead in ((ref5.ref_assemble_split_reads, ()), (H.dh_assemble_split_reads, (ctxh,))):
        so = np.zeros((n, 13), np.int32); srq = np.zeros(n, np.float32); co = np.zeros((n, 2048), np.uint8); cl = np.zeros(n, np.int32)
        al = np.zeros((n, 4096), np.uint8); all_ = np.zeros(n, np.int32)
        rc = fn(*lead, _p(d["contig"]), _p(d["coff"]), _p(d["clen"]), 2, _p(d["rec"]), nrec, _p(d["cig"]), _p(d["reads"]), _p(d["store"]), len(d["store"]), _p(d["sv"]), n,
                max_per_sv, 1, 2, C.c_float(0.95), 13, 1000, 100, _p(so), _p(srq), _p(co), 2048, _p(cl), _p(al), 4096, _p(all_))
        assert rc == 0, rc
        outs.append((so.copy(), srq.copy(), [co[i, :cl[i]].tobytes() for i in range(n)], [al[i, :all_[i]].tobytes() for i in range(n)]))
    e, g = outs
    for i in range(n):
        assert g[2][i] == e[2][i], (i, d["sv"][i].tolist(), len(g[2][i]), len(e[2][i]))
        assert g[0][i].tolist() == e[0][i].tolist(), (i, d["sv"][i].tolist(), g[0][i].tolist(), e[0][i].tolist())
        assert g[3][i] == e[3][i]
    assert np.array_equal(e[1].view(np.uint32), g[1].view(np.uint32))
    big = (d["sv"][:, 4] >= 5) == big_tra
    assert (e[0][big, 8] > 0).sum() >= big.sum() // 3     # most large clusters give a precise call


# ---- whole program: `delly sr -p 200` on a 120x sample --------------------------------------------------------------------

def test_high_coverage_max_reads_bcf_identical(binding_large, tmp_path):
    prefix = str(tmp_path / "hc")
    _run([os.path.join(ROOT, "delly_b200", "bin", "simbam"), "--out", prefix, "--genome-len", "400000", "--contigs", "2", "--n-sv", "12", "--cov", "120",
          "--types", "DEL,DUP,INV", "--seed", "7"])
    common = ["sr", "-p", "200", "-g", prefix + ".fa"]
    ref_out, our_out = str(tmp_path / "ref.bcf"), str(tmp_path / "ours.bcf")
    _run([DELLY_REF] + common + ["-o", ref_out, prefix + ".bam"])
    r = _run([binding_large] + common + ["-o", our_out, prefix + ".bam"])
    assert "read cluster(s)" not in r.stderr
    assert _inflate(ref_out) == _inflate(our_out), "BCF streams differ"
    assert open(ref_out + ".csi", "rb").read() == open(our_out + ".csi", "rb").read()
    vcf = _run([DELLY_REF] + common + [prefix + ".bam"]).stdout
    sr = [int(x) for x in re.findall(r";SR=(\d+);", vcf)]
    assert sr and max(sr) > 32
