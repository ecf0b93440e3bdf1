"""The SV-read dump (`-d reads.gz`) of `delly_b200 sr|lr` against the reference's own drivers (oracle/_ref/delly_ref): the same arguments and
path strings to both, then (a) the inflated dumps are identical byte for byte, (b) the BCF with -d equals the reference's and the one
written without -d, (c) the dump holds what the case is about.

[gpu]            the real binary (delly_b200/bin/delly_b200) on an H100: the reads are classified by the batched device alignments.
[edlib-standin]  the CPU suite: the same binding source with the alignment entry points forwarded to the reference's own functions."""
import collections
import gzip
import itertools
import os
import subprocess

import pytest

from test_bcf_parity import DELLY_REF, EX, ROOT, _inflate, _run, _standin_binary

SIMBAM = os.path.join(ROOT, "delly_b200", "bin", "simbam")
MEI = ["--mei", os.path.join(ROOT, "delly_b200", "data", "_mei_templates.fa")]


@pytest.fixture(params=[pytest.param("gpu", marks=pytest.mark.gpu), "edlib-standin"])
def binding(request):
    assert os.path.exists(DELLY_REF) and os.path.isdir(EX), "oracle/_ref/delly_ref or oracle/_ref/example missing: run __graft_entry__.build() where /root/reference exists"
    if request.param == "gpu":
        exe = os.path.join(ROOT, "delly_b200", "bin", "delly_b200")
        assert os.path.exists(exe), "delly_b200/bin/delly_b200 not built"
        return [exe]
    return [_standin_binary()] + MEI


def _dump_pair(binding, mode, bams, tmp_path, genome=None, extra=()):
    """Runs both programs with -d and ours once more without it. Returns the dump lines, or None when neither program created the file."""
    ref_bcf, our_bcf, plain_bcf = (str(tmp_path / f"{n}.bcf") for n in ("ref", "ours", "plain"))
    ref_dump, our_dump = str(tmp_path / "ref.reads.gz"), str(tmp_path / "ours.reads.gz")
    common = ["-g", genome or os.path.join(EX, "ref.fa")] + list(extra)
    mei = binding[1:] if mode == "lr" else []
    _run([DELLY_REF, mode] + common + ["-o", ref_bcf, "-d", ref_dump] + bams)
    _run([binding[0], mode] + mei + common + ["-o", our_bcf, "-d", our_dump] + bams)
    _run([binding[0], mode] + mei + common + ["-o", plain_bcf] + bams)
    a = _inflate(ref_bcf)
    assert a == _inflate(our_bcf), "BCF with -d differs from the reference's"
    assert a == _inflate(plain_bcf), "BCF with -d differs from the BCF without it"
    assert os.path.exists(ref_dump) == os.path.exists(our_dump), "only one program created the dump"
    if not os.path.exists(ref_dump):
        return None
    d = gzip.open(ref_dump, "rb").read()
    assert d == gzip.open(our_dump, "rb").read(), "inflated dumps differ"
    return d.decode().splitlines()


def _rows(lines):
    return [l.split("\t") for l in lines[1:]]


def _link(tmp_path, bam, name):
    """the same alignments under another path, so that the dump's bam column tells the files apart"""
    p = str(tmp_path / name)
    os.symlink(bam, p)
    os.symlink(bam + ".bai", p + ".bai")
    return p


def _sites(tmp_path, mode):
    sites = str(tmp_path / "sites.bcf")
    _run([DELLY_REF, mode, "-g", os.path.join(EX, "ref.fa"), "-o", sites, os.path.join(EX, mode + ".bam")])
    return sites


def test_sr_discovery_dump(binding, tmp_path):
    lines = _dump_pair(binding, "sr", [os.path.join(EX, "sr.bam")], tmp_path)
    assert lines[0] == "#svid\tbam\tqname\tchr\tpos\tmatechr\tmatepos\tmapq\ttype"
    types = {r[8] for r in _rows(lines) if r[0] == "DEL00000000"}
    assert types == {"SR", "PE"}


def test_lr_discovery_dump(binding, tmp_path):
    lines = _dump_pair(binding, "lr", [os.path.join(EX, "lr.bam")], tmp_path)
    assert lines[0] == "#svid\tbam\tqname\tchr\tpos\tmapq\ttype"
    assert any(r[0] == "DEL00000000" and r[6] == "SR" for r in _rows(lines))


@pytest.mark.parametrize("mode", ["sr", "lr"])
def test_genotyping_mode_dump(binding, tmp_path, mode):
    """-v: the sites of the reference's discovery run genotyped again"""
    lines = _dump_pair(binding, mode, [os.path.join(EX, mode + ".bam")], tmp_path, extra=["-v", _sites(tmp_path, mode)])
    assert len(lines) > 5


def test_sr_two_samples_file_major(binding, tmp_path):
    bams = [os.path.join(EX, "sr.bam"), _link(tmp_path, os.path.join(EX, "sr.bam"), "other.bam")]
    rows = _rows(_dump_pair(binding, "sr", bams, tmp_path))
    files = [r[1] for r in rows]
    assert files == sorted(files, key=bams.index) and set(files) == set(bams)


def test_lr_two_samples_contig_major(binding, tmp_path):
    """three contigs, two files: the long-read lines run contig by contig, and file by file within a contig"""
    pre = str(tmp_path / "lrs")
    _run([SIMBAM, "--out", pre, "--genome-len", "600000", "--contigs", "3", "--n-sv", "30", "--cov", "12", "--read-len", "3000", "--isize", "8000",
          "--isd", "300", "--err", "0.01", "--seed", "7", "--types", "DEL,DUP,INV", "--threads", "4"])
    bams = [pre + ".bam", _link(tmp_path, pre + ".bam", "other.bam")]
    rows = _rows(_dump_pair(binding, "lr", bams, tmp_path, genome=pre + ".fa"))
    blocks = [k for k, _ in itertools.groupby((r[3], r[1]) for r in rows)]
    contigs = sorted({r[3] for r in rows})
    assert len(contigs) == 3
    assert blocks == [(c, b) for c in contigs for b in bams]


@pytest.mark.parametrize("mode", ["discovery", "genotyping"])
def test_sr_exclude_intervals_dump(binding, tmp_path, mode):
    """-x: the genotyping pass reads whole contigs, so the dump names records outside the valid regions too"""
    fai = [l.split("\t") for l in open(os.path.join(EX, "ref.fa.fai"))]
    name, length = fai[0][0], int(fai[0][1])
    ex = tmp_path / "exclude.tsv"
    ex.write_text(f"{name}\t{length // 3}\t{length // 3 + length // 8}\n{name}\t{length - 2000}\t{length - 500}\n")
    extra = ["-x", str(ex)] + (["-v", _sites(tmp_path, "sr")] if mode == "genotyping" else [])
    lines = _dump_pair(binding, "sr", [os.path.join(EX, "sr.bam")], tmp_path, extra=extra)
    assert len(lines) > 5


def test_sr_synthetic_sample_with_read_cap(binding, tmp_path):
    """several contigs, DEL / DUP / INV, two files and -a 5: the per-SV cap drops ALT reads, so at most five SR lines per SV and file"""
    pre = str(tmp_path / "sim")
    _run([SIMBAM, "--out", pre, "--genome-len", "3000000", "--contigs", "3", "--n-sv", "300", "--cov", "30", "--seed", "5", "--types", "DEL,DUP,INV",
          "--threads", "4"])
    bams = [pre + ".bam", _link(tmp_path, pre + ".bam", "other.bam")]
    rows = _rows(_dump_pair(binding, "sr", bams, tmp_path, genome=pre + ".fa", extra=["-a", "5"]))
    assert len(rows) > 5000
    assert {r[8] for r in rows} == {"SR", "PE"}
    assert {r[0][:3] for r in rows} == {"DEL", "DUP", "INV"} and len({r[0] for r in rows}) > 200
    sr = collections.Counter((r[0], r[1]) for r in rows if r[8] == "SR")
    assert max(sr.values()) == 5


@pytest.mark.parametrize("mode", ["sr", "lr"])
def test_empty_call_set_creates_no_dump(binding, tmp_path, mode):
    """-t BND finds nothing in the example: the reference never reaches the code that opens the dump (annotateCoverage, genotypeLR)"""
    assert _dump_pair(binding, mode, [os.path.join(EX, mode + ".bam")], tmp_path, extra=["-t", "BND"]) is None


def test_dump_refused_over_several_ranks(binding, tmp_path):
    dump = str(tmp_path / "reads.gz")
    r = subprocess.run([binding[0], "sr", "-g", os.path.join(EX, "ref.fa"), "-d", dump, "--rank", "0", "--nranks", "2", "--comm-file", str(tmp_path / "id"),
                        os.path.join(EX, "sr.bam")], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "-d" in r.stderr and "--nranks" in r.stderr
    assert not os.path.exists(dump) and not os.path.exists(str(tmp_path / "id"))


def test_unwritable_dump_path_fails(binding, tmp_path):
    r = subprocess.run([binding[0], "sr", "-g", os.path.join(EX, "ref.fa"), "-o", str(tmp_path / "o.bcf"), "-d", str(tmp_path / "missing" / "reads.gz"),
                        os.path.join(EX, "sr.bam")], capture_output=True, text=True)
    assert r.returncode != 0 and "dump" in r.stderr
