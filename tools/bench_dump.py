#!/usr/bin/env python
"""What the SV-read dump (`-d`) costs: `delly_b200 sr` with and without -d on the pipeline sample of bench.py (simbam: 8 Mbp in 4 contigs,
30x 150 bp pairs, 1600 planted het / hom DEL / DUP / INV), next to the reference's own drivers (oracle/_ref/delly_ref -h <all host threads>)
with and without -d. When it dumps, the reference aligns the junction reads of its genotyping pass one at a time on one thread
(src/coverage.h:517); delly_b200 keeps its batched device alignments and only adds the bookkeeping and the gzip stream.

  ours_s / ours_dump_s   wall clock of the process, three runs each, alternated (after one warm-up run of each)
  stages_ms              the --timing breakdown of the fastest run of each
  reference_s / reference_dump_s   one run each
  dump_lines             lines of the inflated dump, header included
  bcf_identical          all four BCFs identical (BGZF inflated, ##fileDate aside); dump_identical: both dumps identical once inflated

Usage: python tools/bench_dump.py [--out FILE]   (one JSON line on stdout, also written to FILE)
"""
import argparse
import gzip
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_info, host_cores  # noqa: E402
from delly_b200 import pipeline_bench as pb  # noqa: E402


def timed(cmd):
    t0 = time.perf_counter()
    r = subprocess.run(cmd, capture_output=True, text=True)
    dt = time.perf_counter() - t0
    if r.returncode != 0:
        raise RuntimeError(f"{cmd[0]} failed: " + r.stderr[-800:])
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    d = tempfile.mkdtemp(prefix="dgpu_dump")
    pre = os.path.join(d, "s")
    cores = host_cores()
    sim = pb.simulate(pre, 8_000_000, 4, 1600, seed=11, threads=min(cores, 16))
    ours = lambda out, timing, dump: pb.ours_cmd(pre, out, timing=timing)[:-1] + (["-d", dump] if dump else []) + [pre + ".bam"]
    runs = {"plain": [], "dump": []}
    for k in ("plain", "dump"):   # warm-up: page cache, CUDA module load
        timed(ours(pre + f".{k}.bcf", None, pre + ".ours.reads.gz" if k == "dump" else None))
    for i in range(args.repeats):
        for k in ("plain", "dump"):
            timing = pre + f".{k}.{i}.json"
            dt = timed(ours(pre + f".{k}.bcf", timing, pre + ".ours.reads.gz" if k == "dump" else None))
            runs[k].append((dt, json.load(open(timing))["stages_ms"]))
    ref_cmd = lambda out, dump: [pb.DELLY_REF, "sr", "-g", pre + ".fa", "-o", out, "-h", str(cores)] + (["-d", dump] if dump else []) + [pre + ".bam"]
    t_ref = timed(ref_cmd(pre + ".ref.bcf", None))
    t_ref_dump = timed(ref_cmd(pre + ".ref.dump.bcf", pre + ".ref.reads.gz"))
    bcfs = [pb.inflate(pre + f) for f in (".plain.bcf", ".dump.bcf", ".ref.bcf", ".ref.dump.bcf")]
    ours_dump = gzip.open(pre + ".ours.reads.gz", "rb").read()
    ref_dump = gzip.open(pre + ".ref.reads.gz", "rb").read()
    best = {k: min(v, key=lambda r: r[0]) for k, v in runs.items()}
    res = {
        "workload": "delly sr discovery + genotyping, simbam 8 Mbp / 4 contigs / 30x / 1600 planted DEL,DUP,INV (seed 11), with and without -d",
        "gpu": gpu_info(0), "simulate": sim, "reference_threads": cores,
        "ours_s": [r[0] for r in runs["plain"]], "ours_dump_s": [r[0] for r in runs["dump"]],
        "stages_ms": best["plain"][1], "stages_ms_dump": best["dump"][1],
        "reference_s": t_ref, "reference_dump_s": t_ref_dump,
        "dump_lines": ours_dump.count(b"\n"), "dump_bytes_gz": os.path.getsize(pre + ".ours.reads.gz"),
        "bcf_identical": all(b == bcfs[0] for b in bcfs), "dump_identical": ours_dump == ref_dump,
        "records": pb.count_records(pre + ".plain.bcf"),
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
