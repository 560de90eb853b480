#!/usr/bin/env python
"""Cost of a contig-sharded index (--indexShards N) on one GPU, at a BASELINE config 2 scale model.

Writes a seeded workload to a scratch directory: a random reference (default 100 Mbp in 16 contigs) and reads drawn from it
(default 20,000 x 10 kb, 1-10 % divergence, either strand). Runs mashmap-b200 -s 5000 --pi 85 on it with --indexShards
1, 2 and 4, all shards on device 0, and reports per N: wall time, the index build, the program's own "time spent mapping
the query" and its device-call seconds (the reads fit one batch, so these are per batch), the index image bytes of every
shard, and whether the PAF equals the unsharded run's byte for byte. Prints one JSON line with the GPU's name and power
limit read in the same run.
usage: shard_perf.py [--ref-bp N] [--contigs N] [--reads N] [--read-len N] [--threads N] [--shards 1,2,4]"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from mashmap_b200 import hostlib, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--ref-bp", type=int, default=100_000_000)
ap.add_argument("--contigs", type=int, default=16)
ap.add_argument("--reads", type=int, default=20_000)
ap.add_argument("--read-len", type=int, default=10_000)
ap.add_argument("--threads", type=int, default=16)
ap.add_argument("--shards", default="1,2,4")
ap.add_argument("--seed", type=int, default=5)
args = ap.parse_args()

OPTS = ["-s", "5000", "--pi", "85"]
wd = tempfile.mkdtemp(prefix="mm_shard_perf_")
rng = np.random.default_rng(args.seed)
clen = args.ref_bp // args.contigs
genome = [synth.random_sequence(clen, rng) for _ in range(args.contigs)]
names = [f"ctg{i}" for i in range(args.contigs)]
reads, rnames = [], []
for i in range(args.reads):
    c, s = int(rng.integers(0, args.contigs)), int(rng.integers(0, clen - args.read_len))
    q = synth.mutate(genome[c][s : s + args.read_len], float(rng.uniform(0.01, 0.10)), rng)
    reads.append(synth.revcomp(q) if rng.random() < 0.5 else q)
    rnames.append(f"r{i}_{names[c]}_{s}")
ref_fa, qry_fa = os.path.join(wd, "ref.fa"), os.path.join(wd, "qry.fa")
synth.write_fasta(ref_fa, names, genome)
synth.write_fasta(qry_fa, rnames, reads)
q_bases = int(sum(len(r) for r in reads))


def number(pat, log):
    m = re.findall(pat, log)
    return float(m[-1]) if m else None


runs, first_paf = {}, None
for n in [int(x) for x in args.shards.split(",")]:
    out = os.path.join(wd, f"shards{n}.paf")
    cmd = [hostlib.CLI_PATH, "-r", ref_fa, "-q", qry_fa, "-t", str(args.threads), "-o", out] + OPTS
    if n > 1:
        cmd += ["--indexShards", str(n)]
    t = time.time()
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    wall = time.time() - t
    assert p.returncode == 0, (cmd, p.stderr[-3000:])
    log = p.stderr
    paf = open(out, "rb").read()
    first_paf = paf if first_paf is None else first_paf
    shard_bytes = [int(b) for b in re.findall(r"shard \d+: \d+ minmers, \d+ lookup keys, (\d+) index bytes", log)]
    runs[str(n)] = {"wall_s": round(wall, 3),
                    "index_build_s": number(r"index built on the device (?:in \d+ shards )?in ([0-9.e+-]+) s", log),
                    "map_s": number(r"time spent mapping the query: ([0-9.e+-]+) sec", log),
                    "device_calls_s": number(r"device calls ([0-9.e+-]+) s", log),
                    "host_tail_s": number(r"host tail ([0-9.e+-]+) s", log),
                    "index_bytes_per_shard": shard_bytes or None,
                    "paf_lines": paf.count(b"\n"), "paf_equals_unsharded": paf == first_paf}
    print(f"--indexShards {n}: {runs[str(n)]}", file=sys.stderr, flush=True)

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                      text=True).stdout.strip().splitlines()
print(json.dumps({"workload": {"ref_bp": args.ref_bp, "contigs": args.contigs, "reads": args.reads, "read_len": args.read_len,
                               "query_bp": q_bases, "options": " ".join(OPTS), "threads": args.threads},
                  "gpu": card[0] if card else None, "runs": runs}))
