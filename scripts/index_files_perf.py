#!/usr/bin/env python
"""--saveIndex and --loadIndex at scale: the index built on the device (the default) against the host builder
(--hostIndex), on the same seeded workload.

Writes to a scratch directory, which is deleted at the end: a random reference (default 1 Gbp in 32 contigs) and a few
thousand reads drawn from it (default 4,000 x 10 kb, 3 % substitutions, either strand), so that building or loading the
index dominates each run. At 1 Gbp each save writes about 4.2 GB (a 1.2 GB PREFIX.index and a 2.9 GB PREFIX.map).
Four CLI runs (-s 5000 --pi 85):
- save_device:  --saveIndex P
- save_host:    --saveIndex Q --hostIndex
- load_device:  --loadIndex P
- load_host:    --loadIndex P --hostIndex
Reports each run's wall time and the phase times it logs. Asserts that P and Q are byte-identical (PREFIX.index and
PREFIX.map) and that the four PAFs are. Prints one JSON line with the GPU's name and power limit read in the same run.
usage: index_files_perf.py [--ref-bp N] [--contigs N] [--reads N] [--read-len N] [--threads N]"""
import argparse
import filecmp
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
from mashmap_b200 import hostlib  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--ref-bp", type=int, default=1_000_000_000)
ap.add_argument("--contigs", type=int, default=32)
ap.add_argument("--reads", type=int, default=4_000)
ap.add_argument("--read-len", type=int, default=10_000)
ap.add_argument("--threads", type=int, default=8)
ap.add_argument("--seed", type=int, default=5)
args = ap.parse_args()

wd = tempfile.mkdtemp(prefix="mm_index_files_perf_")
try:
    rng = np.random.default_rng(args.seed)
    ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
    COMP = np.zeros(256, dtype=np.uint8)
    for a, b in zip(b"ACGT", b"TGCA"):
        COMP[a] = b
    clen = args.ref_bp // args.contigs
    genome = [ACGT[rng.integers(0, 4, clen)] for _ in range(args.contigs)]
    ref, qry = os.path.join(wd, "ref.fa"), os.path.join(wd, "reads.fa")
    with open(ref, "wb") as f:
        for i, g in enumerate(genome):
            body = g.tobytes()
            f.write(b">ctg%d\n" % i + b"\n".join(body[o : o + 80] for o in range(0, len(body), 80)) + b"\n")
    with open(qry, "wb") as f:
        for i in range(args.reads):
            c, s = int(rng.integers(0, args.contigs)), int(rng.integers(0, clen - args.read_len))
            q = genome[c][s : s + args.read_len].copy()
            sub = rng.random(args.read_len) < 0.03
            q[sub] = ACGT[rng.integers(0, 4, int(sub.sum()))]
            seq = COMP[q[::-1]] if rng.random() < 0.5 else q
            f.write(b">r%d_ctg%d_%d\n" % (i, c, s) + seq.tobytes() + b"\n")
    del genome

    def number(pat, log):
        m = re.findall(pat, log)
        return float(m[-1]) if m else None

    P, Q = os.path.join(wd, "dev"), os.path.join(wd, "host")
    runs, first = {}, None
    for mode, extra in (("save_device", ["--saveIndex", P]), ("save_host", ["--saveIndex", Q, "--hostIndex"]),
                        ("load_device", ["--loadIndex", P]), ("load_host", ["--loadIndex", P, "--hostIndex"])):
        out = os.path.join(wd, f"{mode}.paf")
        t0 = time.perf_counter()
        p = subprocess.run([hostlib.CLI_PATH, "-r", ref, "-q", qry, "-s", "5000", "--pi", "85", "-t", str(args.threads), "-o", out] + extra,
                           capture_output=True, text=True)
        wall = time.perf_counter() - t0
        assert p.returncode == 0, p.stderr[-3000:]
        paf = open(out, "rb").read()
        first = paf if first is None else first
        assert paf == first, f"{mode}: PAF differs from the first run's"
        log = p.stderr
        runs[mode] = {
            "wall_s": round(wall, 2),
            "device_build_s": number(r"index built on the device in ([0-9.e+-]+) s", log),
            "device_load_build_s": number(r"index built on the device from the \d+ records of .* in ([0-9.e+-]+) s", log),
            "device_save_s": number(r"index saved to .* in ([0-9.e+-]+) s", log),
            "host_lookup_s": number(r"lookup index \+ frequency filter in ([0-9.e+-]+) s", log),
            "minmers_before_filter": number(r"minmer windows picked from reference = (\d+)", log),
            "paf_lines": paf.count(b"\n"),
        }
        if mode == "save_host":
            for ext in (".index", ".map"):
                assert filecmp.cmp(P + ext, Q + ext, shallow=False), f"{ext}: the device's and the host's saves differ"
            index_bytes = {ext: os.path.getsize(P + ext) for ext in (".index", ".map")}
            for ext in (".index", ".map"):
                os.remove(Q + ext)

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    gpu = smi.stdout.strip().split("\n")[0] if smi.returncode == 0 else "unknown"
    print(json.dumps({
        "gpu": gpu, "host_threads": args.threads, "reference_bp": args.ref_bp, "contigs": args.contigs, "reads": args.reads,
        "read_len": args.read_len, "index_file_bytes": index_bytes, "runs": runs, "saves_identical": True, "paf_identical": True,
    }))
finally:
    shutil.rmtree(wd, ignore_errors=True)
