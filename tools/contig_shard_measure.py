"""What one rank of `delly_b200 sr --shard-by contig` (or `lr` with --lr) reads, holds and sends, on a multi-contig synthetic sample (tools/simbam.cpp).

For N = 1, 2, 4, 8 every rank's share is read alone (`--read-share-only`: the rank's contigs through the BAM index, then stop): the records
it holds, its peak resident memory and its `read_bam` wall time. With --exchange, the complete single-process contig-sharded call runs as
well (it needs the device) and reports the bytes each stage hands to the exchange; at one rank that is every contig's logs, which N ranks
send once each, by the contig's owner (the sample has no inter-chromosomal pairs, so no mate-table entries travel either way).

    python tools/contig_shard_measure.py [--genome-len 24000000] [--cov 30] [--exchange] [--out result.json]
    python tools/contig_shard_measure.py --lr [--read-len 5000] [--cov 20] ...   # long reads: `delly_b200 lr`, multi-kb reads

Prints one JSON object. Numbers from a run on a shared host vary with its load; the records and bytes do not."""
import argparse
import json
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "delly_b200", "bin")


def _timing(path, nranks, rank):
    with open(path + ("." + str(rank) if nranks > 1 else "")) as f:
        return json.load(f)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--genome-len", type=int, default=24_000_000)
    ap.add_argument("--contigs", type=int, default=24)
    ap.add_argument("--cov", type=float, default=None, help="coverage (default 30 for sr, 20 for --lr)")
    ap.add_argument("--lr", action="store_true", help="long reads: simbam reads of --read-len bases, `delly_b200 lr`")
    ap.add_argument("--read-len", type=int, default=5000, help="read length of --lr")
    ap.add_argument("--ranks", default="1,2,4,8")
    ap.add_argument("--io-threads", type=int, default=8)
    ap.add_argument("--exchange", action="store_true", help="also run the complete call at one rank (needs the device) for the exchange sizes")
    ap.add_argument("--out", help="also write the JSON object to this file")
    a = ap.parse_args()
    if a.cov is None:
        a.cov = 20 if a.lr else 30
    with tempfile.TemporaryDirectory() as tmp:
        sim = os.path.join(tmp, "sim")
        reads = ["--read-len", str(a.read_len), "--isize", str(3 * a.read_len), "--isd", "300", "--err", "0.01"] if a.lr else []
        subprocess.run([os.path.join(BIN, "simbam"), "--out", sim, "--contigs", str(a.contigs), "--genome-len", str(a.genome_len), "--cov", str(a.cov),
                        "--types", "DEL,DUP,INV", "--n-sv", "400"] + reads, check=True, capture_output=True)
        base = [os.path.join(BIN, "delly_b200"), "lr" if a.lr else "sr", "--shard-by", "contig", "--io-threads", str(a.io_threads), "-g", sim + ".fa"]
        res = {"sample": {"mode": "lr" if a.lr else "sr", "contigs": a.contigs, "genome_len": a.genome_len, "cov": a.cov, "read_len": a.read_len if a.lr else None,
                          "bam_bytes": os.path.getsize(sim + ".bam")}, "shares": {}}
        for n in [int(x) for x in a.ranks.split(",")]:
            rows = []
            for r in range(n):
                t = os.path.join(tmp, "t%d" % n)
                subprocess.run(base + ["--nranks", str(n), "--rank", str(r), "--read-share-only", "--timing", t, sim + ".bam"], check=True, capture_output=True)
                j = _timing(t, n, r)
                rows.append({"rank": r, "records": j["records"], "peak_rss_mb": round(j["peak_rss_kb"] / 1024, 1), "read_bam_ms": round(j["stages_ms"]["read_bam"], 1)})
            res["shares"][str(n)] = rows
        if a.exchange:
            t = os.path.join(tmp, "full")
            subprocess.run(base + ["--timing", t, "-o", os.path.join(tmp, "calls.bcf"), sim + ".bam"], check=True, capture_output=True)
            j = _timing(t, 1, 0)
            res["exchange_bytes_by_stage"] = j["sent_bytes"]
            res["exchange_bytes_total"] = sum(j["sent_bytes"].values())
            res["svs"] = j["svs"]
    out = json.dumps(res)
    print(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
