#!/usr/bin/env python
"""FASTQ input at full scale: mm_fastq_cut on one window of reads, and the CLI on FASTQ parsed on the device (plain and
BGZF), on the same FASTQ files through the line reader (MM_SERIAL_INPUT=1, the only path before FASTQ was parsed on the
device), and on the same reads as plain FASTA.

Writes a seeded workload to a scratch directory: a random reference (default 1 Gbp in 32 contigs) and reads drawn from it
(default 200,000 x 10 kb, 3 % substitutions, either strand) with a quality line each, as plain FASTQ, as BGZF FASTQ at zlib
level 6 (bgzip's default, compressed on every host thread) and as plain FASTA. Reports:
- mm_fastq_cut on one window of the plain FASTQ text (--window-mb, after a warm-up cut of the same window): its kernels'
  event time and the whole call, and GB/s of text over each;
- for each of the five inputs: the CLI's wall time and its "input read and handed over" time;
- that all five PAFs are byte-identical (asserted).
Prints one JSON line with the GPU's name and power limit read in the same run.
usage: fastq_perf.py [--ref-bp N] [--contigs N] [--reads N] [--read-len N] [--threads N] [--window-mb N]"""
import argparse
import concurrent.futures as cf
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bgzf_data as B  # noqa: E402
from mashmap_b200 import capi, hostlib  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--ref-bp", type=int, default=1_000_000_000)
ap.add_argument("--contigs", type=int, default=32)
ap.add_argument("--reads", type=int, default=200_000)
ap.add_argument("--read-len", type=int, default=10_000)
ap.add_argument("--threads", type=int, default=os.cpu_count())
ap.add_argument("--window-mb", type=int, default=512)
ap.add_argument("--seed", type=int, default=5)
args = ap.parse_args()

HOST_THREADS = os.cpu_count()
wd = tempfile.mkdtemp(prefix="mm_fastq_perf_")
rng = np.random.default_rng(args.seed)
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = np.zeros(256, dtype=np.uint8)
for a, b in zip(b"ACGT", b"TGCA"):
    COMP[a] = b
QUAL = np.frombuffer(b"!#+5?I", dtype=np.uint8)

clen = args.ref_bp // args.contigs
genome = [ACGT[rng.integers(0, 4, clen)] for _ in range(args.contigs)]
with open(os.path.join(wd, "ref.fa"), "wb") as f:
    for i, g in enumerate(genome):
        body = g.tobytes()
        f.write(b">ctg%d\n" % i + b"\n".join(body[o : o + 80] for o in range(0, len(body), 80)) + b"\n")
fa, fq = [], []
for i in range(args.reads):
    c, s = int(rng.integers(0, args.contigs)), int(rng.integers(0, clen - args.read_len))
    q = genome[c][s : s + args.read_len].copy()
    sub = rng.random(args.read_len) < 0.03
    q[sub] = ACGT[rng.integers(0, 4, int(sub.sum()))]
    seq = (COMP[q[::-1]] if rng.random() < 0.5 else q).tobytes()
    name = b"r%d_ctg%d_%d" % (i, c, s)
    fa.append(b">" + name + b"\n" + seq + b"\n")
    fq.append(b"@" + name + b" runid=x ch=1\n" + seq + b"\n+\n" + QUAL[rng.integers(0, len(QUAL), len(seq))].tobytes() + b"\n")
del genome
fq_text = b"".join(fq)
paths = {"ref": os.path.join(wd, "ref.fa"), "fa": os.path.join(wd, "reads.fa"), "fq": os.path.join(wd, "reads.fq"),
         "fq_bgzf": os.path.join(wd, "reads.fq.gz")}
with open(paths["fa"], "wb") as f:
    f.write(b"".join(fa))
with open(paths["fq"], "wb") as f:
    f.write(fq_text)
with cf.ThreadPoolExecutor(HOST_THREADS) as ex:
    members = list(ex.map(lambda o: B.member(fq_text[o : o + B.BLOCK], 6), range(0, len(fq_text), B.BLOCK), chunksize=64))
with open(paths["fq_bgzf"], "wb") as f:
    f.write(b"".join(members) + B.EOF_MARKER)
bgzf_bytes = sum(len(m) for m in members)
del fa, fq, members

# one window of whole records, cut three times: the first two warm up the kernels and size the buffers (a cut's results
# go to one of two sets of pinned buffers, alternately), the third is timed
w = min(len(fq_text), args.window_mb << 20)
w = fq_text.rfind(b"\n@", 0, w) + 1 if w < len(fq_text) else w
window = fq_text[:w]
parser = capi.FastqParser(0)
n_rec = 0
for _ in range(3):
    parser.append_text(window)
    t0 = time.perf_counter()
    got = parser.cut(1)
    cut_wall = time.perf_counter() - t0
    n_rec = len(got["names"])
kernel_ms, call_ms = parser.last_ms()
assert got["consumed"] == len(window) and n_rec == window.count(b"\n@") + 1
parser.close()
del fq_text, window, got


def number(pat, log):
    m = re.findall(pat, log)
    return float(m[-1]) if m else None


cli, first = {}, None
for mode, qry, env in (("fastq_device", paths["fq"], None), ("fastq_bgzf_device", paths["fq_bgzf"], None),
                       ("fastq_line_reader", paths["fq"], {"MM_SERIAL_INPUT": "1"}),
                       ("fastq_bgzf_line_reader", paths["fq_bgzf"], {"MM_SERIAL_INPUT": "1"}),
                       ("fasta", paths["fa"], None)):
    out = os.path.join(wd, f"{mode}.paf")
    t0 = time.perf_counter()
    p = subprocess.run([hostlib.CLI_PATH, "-r", paths["ref"], "-q", qry, "-s", "5000", "--pi", "85", "-t", str(args.threads),
                        "-o", out], capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    wall = time.perf_counter() - t0
    assert p.returncode == 0, p.stderr[-3000:]
    paf = open(out, "rb").read()
    first = paf if first is None else first
    assert paf == first, f"{mode}: PAF differs from the first run's"
    cli[mode] = {"wall_s": round(wall, 2), "input_read_s": number(r"input read and handed over in ([0-9.e+-]+) s", p.stderr),
                 "windows": number(r"FASTQ, parsed on device \d+ in (\d+) windows", p.stderr), "paf_lines": paf.count(b"\n")}

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
gpu = smi.stdout.strip().split("\n")[0] if smi.returncode == 0 else "unknown"
print(json.dumps({
    "gpu": gpu, "host_threads": HOST_THREADS,
    "reference_bp": args.ref_bp, "contigs": args.contigs, "reads": args.reads, "read_len": args.read_len,
    "query_fastq_bytes": os.path.getsize(paths["fq"]), "query_fastq_bgzf_bytes": bgzf_bytes,
    "cut": {"window_bytes": w, "records": n_rec, "kernel_ms": round(kernel_ms, 2), "call_ms": round(call_ms, 2),
            "call_wall_s": round(cut_wall, 3), "kernel_GBps_text": round(w / kernel_ms / 1e6, 2),
            "call_GBps_text": round(w / call_ms / 1e6, 2)},
    "cli": cli, "paf_identical": True,
}))
shutil.rmtree(wd, ignore_errors=True)
