"""Times `delly_b200 sr` over N ranks two ways on the pipeline sample of `bench.py --gpus N` (a simbam sample, 24 Mbp in 8 contigs, 4800 SVs,
30x): N processes exchanging over NCCL (`--rank r --nranks N --comm-file`, one per device) and one process with `--devices` over the same
devices. Each is timed with a host clock around the whole program (all N processes: from the first start to the last exit), with the
`--timing` stage breakdown of every rank; the two BCFs must be identical (BGZF inflated, ##fileDate aside), and a single-rank run on the first
device gives the baseline. Prints one JSON line, with the name and power limit of every card used, read in the same run.

    python tools/bench_devices.py --devices 0,1 [--shard-by svs|contig|both] [--repeats 2] [--genome-len 24000000 --contigs 8 --n-sv 4800]

NCCL runs one rank per device: with a repeated index (`--devices 0,0`) the N-process arm is skipped and reported as not measured."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from delly_b200 import pipeline_bench as pb  # noqa: E402

EXE = os.path.join(pb.BIN, "delly_b200")


def card(index):
    """name and power limit of one card, read now (nvidia-smi query only)"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True,
                           timeout=30)
        name, watts = [x.strip() for x in r.stdout.strip().split(",")]
        return {"device": index, "name": name, "power_limit_w": float(watts)}
    except Exception as e:  # noqa: BLE001
        return {"device": index, "error": repr(e)}


def stages(prefix, n):
    out = []
    for r in range(n):
        p = f"{prefix}.{r}" if n > 1 else prefix
        out.append(json.load(open(p)) if os.path.exists(p) else None)
    return out


def run_processes(pre, out, devices, shard, timing):
    """N rank processes over NCCL; wall = first start to last exit"""
    comm = out + ".ncclid"
    if os.path.exists(comm):
        os.remove(comm)
    n = len(devices)
    t0 = time.perf_counter()
    procs = [subprocess.Popen([EXE, "sr", "-g", pre + ".fa", "-o", out, "--device", str(d), "--rank", str(r), "--nranks", str(n), "--comm-file", comm,
                               "--shard-by", shard, "--timing", timing, pre + ".bam"], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True)
             for r, d in enumerate(devices)]
    errs = [p.communicate()[1] for p in procs]
    wall = time.perf_counter() - t0
    for r, p in enumerate(procs):
        if p.returncode != 0:
            raise RuntimeError(f"rank {r} failed: " + errs[r][-800:])
    return wall, stages(timing, n)


def run_devices(pre, out, devices, shard, timing):
    n = len(devices)
    t0 = time.perf_counter()
    r = subprocess.run([EXE, "sr", "-g", pre + ".fa", "-o", out, "--devices", ",".join(map(str, devices)), "--shard-by", shard, "--timing", timing,
                        pre + ".bam"], capture_output=True, text=True)
    wall = time.perf_counter() - t0
    if r.returncode != 0:
        raise RuntimeError("--devices run failed: " + r.stderr[-800:])
    return wall, stages(timing, n)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--devices", default="0,1")
    ap.add_argument("--shard-by", default="both", choices=["svs", "contig", "both"])
    ap.add_argument("--repeats", type=int, default=2, help="runs per arm, alternated; every wall time is reported")
    ap.add_argument("--genome-len", type=int, default=24_000_000)
    ap.add_argument("--contigs", type=int, default=8)
    ap.add_argument("--n-sv", type=int, default=4800)
    a = ap.parse_args()
    devices = [int(x) for x in a.devices.split(",")]
    n = len(devices)
    nccl_ok = len(set(devices)) == n and n > 1
    d = tempfile.mkdtemp(prefix="dgpu_devices")
    pre = os.path.join(d, "s")
    res = {"devices": devices, "cards": [card(i) for i in sorted(set(devices))],
           "sample": {"genome_len": a.genome_len, "contigs": a.contigs, "n_sv": a.n_sv, "cov": 30},
           "simulate": pb.simulate(pre, a.genome_len, a.contigs, a.n_sv, seed=11, threads=min(os.cpu_count() or 1, 16))}
    one = pre + ".n1.bcf"
    pb.run_ours(pre, one, device=devices[0])   # warm-up: page cache, CUDA module load
    base = [pb.run_ours(pre, one, device=devices[0], timing=pre + ".n1.json") for _ in range(a.repeats)]
    res["single_rank"] = {"wall_s": [b[0] for b in base], "stages_ms": base[-1][1]["stages_ms"] if base[-1][1] else None}
    ref = pb.inflate(one)
    for shard in (["svs", "contig"] if a.shard_by == "both" else [a.shard_by]):
        arm = {"processes": {"wall_s": [], "ranks": None} if nccl_ok else "not measured: NCCL runs one rank per device",
               "devices": {"wall_s": [], "ranks": None}}
        for k in range(a.repeats):
            if nccl_ok:
                out = pre + f".{shard}.proc.bcf"
                wall, st = run_processes(pre, out, devices, shard, pre + f".{shard}.proc.t")
                arm["processes"]["wall_s"].append(wall)
                arm["processes"]["ranks"] = st
                arm["processes"]["bcf_identical_to_single_rank"] = pb.inflate(out) == ref
            out = pre + f".{shard}.dev.bcf"
            wall, st = run_devices(pre, out, devices, shard, pre + f".{shard}.dev.t")
            arm["devices"]["wall_s"].append(wall)
            arm["devices"]["ranks"] = st
            arm["devices"]["bcf_identical_to_single_rank"] = pb.inflate(out) == ref
        if nccl_ok:
            arm["bcfs_identical"] = pb.inflate(pre + f".{shard}.proc.bcf") == pb.inflate(pre + f".{shard}.dev.bcf")
        res[shard] = arm
    res["records"] = pb.count_records(one)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
