#!/usr/bin/env python
"""Queries mapped whole (--noSplit, one fragment longer than a segment: windowLen > 0) on one GPU, against the reference.

Writes a seeded workload to a scratch directory: a random reference (default 200 Mbp in 8 contigs) and queries drawn
from it with 1-10 % divergence (substitutions / insertions / deletions 4:3:3; either strand): 2,000 x 100 kb and 100 x
1 Mbp by default. Then
  * mashmap-b200 -s 5000 --pi 85 --noSplit end to end (wall time and the program's own "time spent mapping the query");
  * the device stages of the same queries through the C ABI (index built on the device, whole queries resident in HBM,
    mm_map_resident; mm_last_stage_ms: sketch incl. the merge of the pieces, L1, L2, first launch -> last kernel end);
  * the unmodified reference (oracle/_ref/mashmap_ref -t 16), where it is built, on a stated subset of the queries (the
    first --ref-100k of the 100 kb and --ref-1m of the 1 Mbp queries), and whether the two programs print the same PAF
    lines for that subset (first 12 columns equal and in the same order, identity within 1e-4).
Prints one JSON line (GPU name and power limit included).
usage: nosplit_perf.py [--ref-bp N] [--n100k N] [--n1m N] [--ref-100k N] [--ref-1m N] [--threads N]"""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
from mashmap_b200 import capi, hostlib, synth  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--ref-bp", type=int, default=200_000_000)
ap.add_argument("--contigs", type=int, default=8)
ap.add_argument("--n100k", type=int, default=2000)
ap.add_argument("--n1m", type=int, default=100)
ap.add_argument("--ref-100k", type=int, default=100, help="100 kb queries in the reference arm's subset")
ap.add_argument("--ref-1m", type=int, default=5, help="1 Mbp queries in the reference arm's subset")
ap.add_argument("--threads", type=int, default=16)
ap.add_argument("--seed", type=int, default=7)
args = ap.parse_args()

REF_BIN = os.path.join(ROOT, "oracle", "_ref", "mashmap_ref")
OPTS = ["-s", "5000", "--pi", "85", "--noSplit"]
wd = tempfile.mkdtemp(prefix="mm_nosplit_perf_")
rng = np.random.default_rng(args.seed)
t0 = time.time()
clen = args.ref_bp // args.contigs
genome = [synth.random_sequence(clen, rng) for _ in range(args.contigs)]
names = [f"ctg{i}" for i in range(args.contigs)]


def draw(n, length, tag):
    out, qn = [], []
    for i in range(n):
        c = int(rng.integers(0, args.contigs))
        s = int(rng.integers(0, clen - length))
        q = synth.mutate(genome[c][s : s + length], float(rng.uniform(0.01, 0.10)), rng)
        if rng.random() < 0.5:
            q = synth.revcomp(q)
        out.append(q)
        qn.append(f"{tag}{i}_{names[c]}_{s}")
    return out, qn


q100, n100 = draw(args.n100k, 100_000, "q100k_")
q1m, n1m = draw(args.n1m, 1_000_000, "q1m_")
queries, qnames = q100 + q1m, n100 + n1m
ref_fa, qry_fa, sub_fa = (os.path.join(wd, f) for f in ("ref.fa", "qry.fa", "qry_subset.fa"))
synth.write_fasta(ref_fa, names, genome)
synth.write_fasta(qry_fa, qnames, queries)
subset = list(range(min(args.ref_100k, args.n100k))) + [args.n100k + i for i in range(min(args.ref_1m, args.n1m))]
synth.write_fasta(sub_fa, [qnames[i] for i in subset], [queries[i] for i in subset])
q_bases = int(sum(len(q) for q in queries))
print(f"workload: {args.ref_bp / 1e6:.0f} Mbp reference, {len(queries)} queries, {q_bases / 1e6:.0f} Mbp, written in "
      f"{time.time() - t0:.0f} s", file=sys.stderr, flush=True)


def run(cmd):
    t = time.time()
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 0, (cmd, p.stderr[-3000:])
    return time.time() - t, p.stderr


def mapping_seconds(log):
    return float([ln for ln in log.splitlines() if "time spent mapping the query" in ln][-1].split(":")[-1].split()[0])


def cli_breakdown(log):
    """the product's own timing lines: device index build, device contexts + pinned buffers, reading the queries and the
    end of the last batch (seconds)"""
    out = {}
    pats = {"index_build_s": r"index built on the device in ([0-9.e+-]+) s", "contexts_s": r"device contexts \+ index upload ([0-9.e+-]+) s",
            "pinned_buffers_s": r"pinned batch buffers ([0-9.e+-]+) s", "input_read_s": r"input read and handed over in ([0-9.e+-]+) s",
            "last_batch_done_s": r"last batch done at ([0-9.e+-]+) s"}
    for k, pat in pats.items():
        m = re.findall(pat, log)
        out[k] = float(m[-1]) if m else None
    return out


# ---- the product, end to end ----
got_paf = os.path.join(wd, "got.paf")
wall, log = run([hostlib.CLI_PATH, "-r", ref_fa, "-q", qry_fa, "-t", str(args.threads), "-o", got_paf] + OPTS)
sketch_size = int([ln for ln in log.splitlines() if "Sketch size = " in ln][-1].split("=")[-1])
result = {"workload": {"ref_bp": args.ref_bp, "queries_100kb": args.n100k, "queries_1mb": args.n1m, "query_bp": q_bases,
                       "divergence": [0.01, 0.10], "options": " ".join(OPTS), "sketch_size": sketch_size},
          "cli": {"wall_s": round(wall, 3), "map_s": mapping_seconds(log), "paf_lines": sum(1 for _ in open(got_paf)),
                  "query_gbp_per_s": round(q_bases / mapping_seconds(log) / 1e9, 4), **cli_breakdown(log)}}

# ---- the device stages of the same queries (C ABI, resident batch) ----
ctx = capi.Context(kmer_size=19, seg_length=5000, sketch_size=sketch_size)
offs = np.zeros(args.contigs + 1, dtype=np.uint64)
offs[1:] = np.cumsum([len(c) for c in genome])
ctx.index_build(np.concatenate(genome), offs)
ctx.tables_upload(hostlib.sketch_cutoffs(sketch_size, 19), hostlib.min_hits_table(sketch_size, 19, 0.85))
qoff = np.zeros(len(queries) + 1, dtype=np.int64)
qoff[1:] = np.cumsum([len(q) for q in queries])
segs = np.zeros(len(queries), dtype=capi.segment_dtype)
segs["offset"] = qoff[:-1]
segs["length"] = [len(q) for q in queries]
segs["seq_counter"] = np.arange(len(queries))
segs["name_id"] = -1
segs["ref_group"] = -1
ctx.batch_upload(np.concatenate(queries), segs)
runs = []
for _ in range(4):
    ctx.map_resident()
    runs.append(ctx.stage_ms())
ms = np.median(np.array(runs[1:]), axis=0)  # the first run allocates the work areas
result["device_ms"] = {"k1_sketch_incl_merge": round(float(ms[0]), 2), "k2_l1": round(float(ms[1]), 2), "k3_l2": round(float(ms[2]), 2),
                       "first_launch_to_last_kernel": round(float(ms[5]), 2), "runs": len(runs) - 1,
                       "query_gbp_per_s": round(q_bases / (float(ms[5]) / 1e3) / 1e9, 3)}
result["diag"] = ctx.diag()
ctx.close()

# ---- the reference on the subset ----
if os.path.exists(REF_BIN):
    sub_bases = int(sum(len(queries[i]) for i in subset))
    ref_paf, got_sub = os.path.join(wd, "ref_sub.paf"), os.path.join(wd, "got_sub.paf")
    rwall, rlog = run([REF_BIN, "-r", ref_fa, "-q", sub_fa, "-t", "16", "-o", ref_paf] + OPTS)
    gwall, glog = run([hostlib.CLI_PATH, "-r", ref_fa, "-q", sub_fa, "-t", str(args.threads), "-o", got_sub] + OPTS)
    ref_rows = [ln.rstrip("\n").split("\t") for ln in open(ref_paf)]
    got_rows = [ln.rstrip("\n").split("\t") for ln in open(got_sub)]
    same = [r[:12] for r in ref_rows] == [g[:12] for g in got_rows] and all(
        abs(float(r[12].split(":")[2]) - float(g[12].split(":")[2])) <= 1e-4 for r, g in zip(ref_rows, got_rows))
    # the subset's lines must also be what the full run printed for those queries
    sub_names = {qnames[i] for i in subset}
    full_rows = [ln.rstrip("\n").split("\t") for ln in open(got_paf)]
    same_full = [g[:12] for g in got_rows] == [f[:12] for f in full_rows if f[0] in sub_names]
    result["reference_subset"] = {"queries_100kb": min(args.ref_100k, args.n100k), "queries_1mb": min(args.ref_1m, args.n1m),
                                  "query_bp": sub_bases, "threads": 16, "wall_s": round(rwall, 3),
                                  "map_s": mapping_seconds(rlog) if "time spent mapping" in rlog else None,
                                  "product_wall_s": round(gwall, 3), "product_map_s": mapping_seconds(glog),
                                  "paf_lines": len(ref_rows), "paf_equal": bool(same),
                                  "subset_lines_equal_full_run": bool(same_full)}
else:
    result["reference_subset"] = None
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
except Exception:
    name, power = None, None
result["gpu"] = {"name": name, "power_limit": power}
print(json.dumps(result))
