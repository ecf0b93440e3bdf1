"""`delly_b200 sr|lr --devices LIST`: every rank a host thread of one process, on its own device and context, the ranks exchanging through
the in-process all-gatherv (host/shard.hpp SimExchange) instead of NCCL. The BCF (inflated, ##fileDate aside) and its CSI index must be
byte-identical to the single-rank run and to the reference's own drivers (oracle/_ref/delly_ref); the option conflicts are refused before
anything is read or written; one rank's failure releases the others.

[gpu]            the real binary on an H100; repeated indices (0,0 / 0,0,0) put several ranks on one GPU, `--devices 0,1` needs two.
[edlib-standin]  the CPU suite: the same binding source with the alignment entry points forwarded to the reference's own functions."""
import json
import os
import subprocess

import pytest

from test_bcf_parity import DELLY_REF, EX, HERE, REFDIR, ROOT, _inflate, _run, _standin_binary, binding  # noqa: F401 (binding: fixture)

SIMBAM = os.path.join(ROOT, "delly_b200", "bin", "simbam")
MEI = ["--mei", os.path.join(ROOT, "delly_b200", "data", "_mei_templates.fa")]

_cache = {}


def _bcf(cmd, out):
    """(inflated BCF, CSI) of one run writing `out`"""
    _run(cmd + ["-o", out])
    return _inflate(out), open(out + ".csi", "rb").read()


def _once(key, make):
    if key not in _cache:
        _cache[key] = make()
    return _cache[key]


def _check(binding, mode, bams, tmp_path, devices, shard, extra=(), genome=None, with_ref=True):
    """--devices against the run without it and against the reference; returns the inflated BCF"""
    common = ["-g", genome or os.path.join(EX, "ref.fa")] + list(extra)
    mei = binding[1:] if mode == "lr" else []
    key = (binding[0], mode, tuple(bams), tuple(common))
    plain = _once(key + ("plain",), lambda: _bcf([binding[0], mode] + mei + common + bams, str(tmp_path / "plain.bcf")))
    ours = _bcf([binding[0], mode] + mei + common + ["--devices", devices, "--shard-by", shard] + bams, str(tmp_path / "devices.bcf"))
    assert len(plain[0]) > 1000
    assert ours[0] == plain[0], "BCF with --devices differs from the single-rank BCF"
    assert ours[1] == plain[1], "CSI with --devices differs from the single-rank CSI"
    if with_ref:
        ref = _once(key + ("ref",), lambda: _bcf([DELLY_REF, mode] + common + bams, str(tmp_path / "ref.bcf")))
        assert ours == ref, "BCF / CSI with --devices differ from the reference's"
    return ours[0]


def _sites(tmp_path, mode):
    sites = str(tmp_path / "sites.bcf")
    _run([DELLY_REF, mode, "-g", os.path.join(EX, "ref.fa"), "-o", sites, os.path.join(EX, mode + ".bam")])
    return sites


def _link(tmp_path, bam, name):
    """the same alignments under another path (a second sample)"""
    p = str(tmp_path / name)
    os.symlink(bam, p)
    os.symlink(bam + ".bai", p + ".bai")
    return p


@pytest.mark.parametrize("shard", ["svs", "contig"])
@pytest.mark.parametrize("devices", ["0,0", "0,0,0"])
@pytest.mark.parametrize("mode", ["sr", "lr"])
def test_example_identical(binding, tmp_path, mode, devices, shard):
    a = _check(binding, mode, [os.path.join(EX, mode + ".bam")], tmp_path, devices, shard)
    assert b"DEL00000000" in a


@pytest.mark.parametrize("shard", ["svs", "contig"])
@pytest.mark.parametrize("mode", ["sr", "lr"])
def test_genotyping_mode_identical(binding, tmp_path, mode, shard):
    """-v: the reference's discovery BCF genotyped again"""
    _check(binding, mode, [os.path.join(EX, mode + ".bam")], tmp_path, "0,0", shard, extra=["-v", _sites(tmp_path, mode)])


@pytest.mark.parametrize("genotyping", [False, True])
@pytest.mark.parametrize("shard", ["svs", "contig"])
def test_sr_exclude_intervals_identical(binding, tmp_path, shard, genotyping):
    """-x: the process reads the valid regions and the whole contigs (svs: once for all ranks)"""
    fai = [l.split("\t") for l in open(os.path.join(EX, "ref.fa.fai"))]
    name, length = fai[0][0], int(fai[0][1])
    ex = tmp_path / "exclude.tsv"
    ex.write_text(f"{name}\t{length // 3}\t{length // 3 + length // 8}\n{name}\t{length - 2000}\t{length - 500}\n")
    extra = ["-x", str(ex)] + (["-v", _sites(tmp_path, "sr")] if genotyping else [])
    _check(binding, "sr", [os.path.join(EX, "sr.bam")], tmp_path, "0,0,0", shard, extra=extra)


@pytest.mark.parametrize("shard", ["svs", "contig"])
@pytest.mark.parametrize("mode", ["sr", "lr"])
def test_two_samples_identical(binding, tmp_path, mode, shard):
    bams = [os.path.join(EX, mode + ".bam"), _link(tmp_path, os.path.join(EX, mode + ".bam"), "other.bam")]
    _check(binding, mode, bams, tmp_path, "0,0", shard)


@pytest.mark.parametrize("mode", ["sr", "lr"])
def test_three_contigs_three_ranks(binding, tmp_path, mode):
    """a synthetic sample with three contigs: under --shard-by contig each of three ranks reads a contig of its own"""
    pre = str(tmp_path / "sim")
    args = ["--genome-len", "600000", "--contigs", "3", "--n-sv", "30", "--cov", "12", "--seed", "7", "--types", "DEL,DUP,INV", "--threads", "4"]
    if mode == "lr":
        args += ["--read-len", "3000", "--isize", "8000", "--isd", "300", "--err", "0.01"]
    _run([SIMBAM, "--out", pre] + args)
    for shard in ("contig", "svs"):
        _check(binding, mode, [pre + ".bam"], tmp_path, "0,0,0", shard, genome=pre + ".fa", with_ref=False)


def test_two_devices_identical(binding, tmp_path, request):
    if request.node.callspec.params["binding"] != "gpu":
        pytest.skip("a second device means nothing to the CPU stand-in")
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    for shard in ("svs", "contig"):
        _check(binding, "sr", [os.path.join(EX, "sr.bam")], tmp_path, "0,1", shard)


REFUSED = {
    "rank": (["--devices", "0,0", "--rank", "0"], "--rank"),
    "nranks": (["--nranks", "2", "--devices", "0,0"], "--nranks"),
    "comm-file": (["--devices", "0,0", "--comm-file", "{tmp}/id"], "--comm-file"),
    "device": (["--devices", "0,0", "--device", "0"], "--device"),
    "dump": (["--devices", "0,0", "-d", "{tmp}/reads.gz"], "-d"),
    "empty": (["--devices", ""], "--devices"),
    "descending": (["--devices", "1-0"], "--devices"),
    "empty-entry": (["--devices", "0,,1"], "--devices"),
}


def _refused(binding, tmp_path, args, name):
    out = tmp_path / "o.bcf"
    args = [a.replace("{tmp}", str(tmp_path)) for a in args]
    r = subprocess.run([binding[0], "sr", "-g", os.path.join(EX, "ref.fa"), "-o", str(out)] + args + [os.path.join(EX, "sr.bam")],
                       capture_output=True, text=True, timeout=60)
    assert r.returncode != 0, r.stderr
    assert name in r.stderr and "--devices" in r.stderr, r.stderr
    assert sorted(os.listdir(tmp_path)) == [], "a refused run created files"


@pytest.mark.parametrize("case", sorted(REFUSED))
def test_refused(binding, tmp_path, case):
    args, name = REFUSED[case]
    _refused(binding, tmp_path, args, name)


def test_device_index_beyond_count_refused(binding, tmp_path, request):
    if request.node.callspec.params["binding"] != "gpu":
        pytest.skip("the stand-in has no device count")
    import torch
    n = torch.cuda.device_count()
    _refused(binding, tmp_path, ["--devices", f"0,{n}"], "--devices")


def _fail_hook_binary():
    """the stand-in binding built with DELLY_B200_FAIL_HOOK: DELLY_B200_FAIL_RANK=r fails rank r's first exchange (a host-side error)"""
    plain = _standin_binary()
    exe = os.path.join(HERE, "standin", "_build", "delly_b200_standin_failhook")
    if not os.path.exists(exe) or os.path.getmtime(exe) < os.path.getmtime(plain):
        pkg = os.path.join(ROOT, "delly_b200")
        hts = os.path.join(REFDIR, "hts")
        r = subprocess.run(["g++", "-std=c++17", "-O2", "-w", "-DDELLY_B200_FAIL_HOOK", "-o", exe, os.path.join(HERE, "standin", "binding_standin.cpp"),
                            "-I" + os.path.join(hts, "include"), "-L" + REFDIR, "-l:libdelly_ref.so", "-L" + pkg, "-l:libdelly_b200.so",
                            "-Wl,-rpath," + REFDIR, "-Wl,-rpath," + pkg, os.path.join(hts, "libhts.a"), "-lz", "-lm", "-lpthread"],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.parametrize("shard", ["svs", "contig"])
@pytest.mark.parametrize("mode", ["sr", "lr"])
def test_failing_rank_releases_the_others(tmp_path, mode, shard):
    """rank 1's first exchange fails while rank 0 runs: the process ends non-zero within the timeout, names rank 1 and writes no BCF"""
    exe = _fail_hook_binary()
    out = tmp_path / "o.bcf"
    env = dict(os.environ, DELLY_B200_FAIL_RANK="1")
    r = subprocess.run([exe, mode] + (MEI if mode == "lr" else []) + ["-g", os.path.join(EX, "ref.fa"), "-o", str(out), "--devices", "0,0,0",
                                                                       "--shard-by", shard, os.path.join(EX, mode + ".bam")],
                       capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode != 0
    assert "rank 1 of 3" in r.stderr, r.stderr
    assert not os.path.exists(out) and not os.path.exists(str(out) + ".csi")


@pytest.mark.parametrize("mode", ["sr", "lr"])
def test_timing_per_rank(binding, tmp_path, mode):
    """--timing with --read-share-only: one file per rank, the ranks' records add up to the single rank's"""
    pre = str(tmp_path / "sim")
    _run([SIMBAM, "--out", pre, "--genome-len", "600000", "--contigs", "3", "--n-sv", "20", "--cov", "8", "--seed", "3", "--types", "DEL", "--threads", "4"])
    mei = binding[1:] if mode == "lr" else []
    common = [binding[0], mode] + mei + ["-g", pre + ".fa", "--shard-by", "contig", "--read-share-only"]
    one = str(tmp_path / "one.json")
    _run(common + ["--timing", one, pre + ".bam"])
    many = str(tmp_path / "many.json")
    _run(common + ["--timing", many, "--devices", "0,0", pre + ".bam"])
    single = json.load(open(one))
    ranks = [json.load(open(f"{many}.{r}")) for r in range(2)]
    assert not os.path.exists(f"{many}.2")
    assert [t["rank"] for t in ranks] == [0, 1] and all(t["nranks"] == 2 for t in ranks)
    assert all(t["records"] > 0 for t in ranks)
    assert sum(t["records"] for t in ranks) == single["records"] > 0
    assert all("peak_rss_kb" in t and "read_bam" in t["stages_ms"] for t in ranks)
