#!/usr/bin/env python
"""BGZF input at full scale: the device inflater against zlib on every host thread, and the CLI on plain FASTA, on BGZF
read through the device, and on BGZF through the line reader (MM_SERIAL_INPUT=1, the only path before BGZF was read on
the device).

Writes a seeded workload to a scratch directory: a random reference (default 1 Gbp in 32 contigs) and reads drawn from it
(default 200,000 x 10 kb, 3 % substitutions, either strand), as plain FASTA and as BGZF at zlib level 6 (bgzip's default),
compressed on every host thread. Reports:
- mm_inflate_blocks on every BGZF block of the reads, after a warm-up call: GB/s of text and of compressed bytes, over the
  inflate kernels' event time and over the whole call (uploads and downloads included);
- zlib inflating the same blocks on every host thread (wall clock);
- for each of the three inputs: the CLI's wall time and its "input read and handed over" time, and whether its PAF is
  byte-identical to the plain FASTA run's.
Prints one JSON line with the GPU's name and power limit read in the same run.
usage: bgzf_perf.py [--ref-bp N] [--contigs N] [--reads N] [--read-len N] [--threads N]"""
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
import zlib

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
ap.add_argument("--seed", type=int, default=5)
args = ap.parse_args()

HOST_THREADS = os.cpu_count()
wd = tempfile.mkdtemp(prefix="mm_bgzf_perf_")
rng = np.random.default_rng(args.seed)
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
COMP = np.zeros(256, dtype=np.uint8)
for a, b in zip(b"ACGT", b"TGCA"):
    COMP[a] = b


def fasta_text(names, seqs, width=80):
    out = []
    for n, s in zip(names, seqs):
        out.append(b">" + n.encode() + b"\n")
        body = s.tobytes()
        out.append(b"\n".join(body[o : o + width] for o in range(0, len(body), width)) + b"\n")
    return b"".join(out)


clen = args.ref_bp // args.contigs
genome = [ACGT[rng.integers(0, 4, clen)] for _ in range(args.contigs)]
ref_text = fasta_text([f"ctg{i}" for i in range(args.contigs)], genome)
reads, rnames = [], []
for i in range(args.reads):
    c, s = int(rng.integers(0, args.contigs)), int(rng.integers(0, clen - args.read_len))
    q = genome[c][s : s + args.read_len].copy()
    sub = rng.random(args.read_len) < 0.03
    q[sub] = ACGT[rng.integers(0, 4, int(sub.sum()))]
    reads.append(COMP[q[::-1]] if rng.random() < 0.5 else q)
    rnames.append(f"r{i}_ctg{c}_{s}")
qry_text = fasta_text(rnames, reads)
del genome, reads


def bgzf_parallel(text):
    pieces = [text[o : o + B.BLOCK] for o in range(0, len(text), B.BLOCK)]
    with cf.ThreadPoolExecutor(HOST_THREADS) as ex:
        members = list(ex.map(lambda t: B.member(t, 6), pieces, chunksize=64))
    return members, pieces


paths = {}
for tag, text in (("ref", ref_text), ("qry", qry_text)):
    fa = os.path.join(wd, f"{tag}.fa")
    with open(fa, "wb") as f:
        f.write(text)
    members, pieces = bgzf_parallel(text)
    gz = fa + ".gz"
    with open(gz, "wb") as f:
        f.write(b"".join(members) + B.EOF_MARKER)
    paths[tag] = (fa, gz)
    if tag == "qry":
        q_members, q_pieces = members, pieces
del ref_text

# the reads' blocks: raw DEFLATE data of every member (header 18 bytes, trailer 8)
datas = [m[18:-8] for m in q_members]
comp = np.frombuffer(b"".join(datas), dtype=np.uint8)
coff = np.zeros(len(datas) + 1, dtype=np.uint64)
coff[1:] = np.cumsum([len(d) for d in datas])
ooff = np.zeros(len(datas) + 1, dtype=np.uint64)
ooff[1:] = np.cumsum([len(p) for p in q_pieces])
crc = np.array([zlib.crc32(p) for p in q_pieces], dtype=np.uint32)
text_bytes, comp_bytes = int(ooff[-1]), int(coff[-1])
pinned = capi.PinnedBuffer(text_bytes)
inf = capi.Inflater(0)
rc, bad, _, err = inf.inflate(comp, coff, ooff, crc, out=pinned.array)  # warm-up
assert rc == 0, err
t0 = time.perf_counter()
rc, bad, _, err = inf.inflate(comp, coff, ooff, crc, out=pinned.array)
call_wall = time.perf_counter() - t0
assert rc == 0, err
kernel_ms, call_ms = inf.last_ms()
assert pinned.array[:text_bytes].tobytes() == qry_text
inf.close()
pinned.free()


def zlib_block(d):
    return len(zlib.decompress(d, -15))


t0 = time.perf_counter()
with cf.ThreadPoolExecutor(HOST_THREADS) as ex:
    n = sum(ex.map(zlib_block, datas, chunksize=64))
zlib_s = time.perf_counter() - t0
assert n == text_bytes
del datas, comp, q_members, q_pieces


def number(pat, log):
    m = re.findall(pat, log)
    return float(m[-1]) if m else None


cli, first = {}, None
for mode, ref, qry, env in (("plain", paths["ref"][0], paths["qry"][0], None),
                            ("bgzf_device", paths["ref"][1], paths["qry"][1], None),
                            ("bgzf_line_reader", paths["ref"][1], paths["qry"][1], {"MM_SERIAL_INPUT": "1"})):
    out = os.path.join(wd, f"{mode}.paf")
    t0 = time.perf_counter()
    p = subprocess.run([hostlib.CLI_PATH, "-r", ref, "-q", qry, "-s", "5000", "--pi", "85", "-t", str(args.threads), "-o", out],
                       capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    wall = time.perf_counter() - t0
    assert p.returncode == 0, p.stderr[-3000:]
    paf = open(out, "rb").read()
    first = paf if first is None else first
    cli[mode] = {"wall_s": round(wall, 2), "input_read_s": number(r"input read and handed over in ([0-9.e+-]+) s", p.stderr),
                 "paf_lines": paf.count(b"\n"), "paf_identical": paf == first}

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
gpu = smi.stdout.strip().split("\n")[0] if smi.returncode == 0 else "unknown"
print(json.dumps({
    "gpu": gpu, "host_threads": HOST_THREADS,
    "reference_bp": args.ref_bp, "contigs": args.contigs, "reads": args.reads, "read_len": args.read_len,
    "query_text_bytes": text_bytes, "query_bgzf_bytes": comp_bytes, "blocks": len(crc),
    "device_inflate": {"kernel_ms": round(kernel_ms, 2), "call_ms": round(call_ms, 2), "call_wall_s": round(call_wall, 3),
                       "kernel_GBps_text": round(text_bytes / kernel_ms / 1e6, 2),
                       "kernel_GBps_compressed": round(comp_bytes / kernel_ms / 1e6, 2),
                       "call_GBps_text": round(text_bytes / call_ms / 1e6, 2)},
    "zlib_all_host_threads": {"s": round(zlib_s, 3), "GBps_text": round(text_bytes / zlib_s / 1e9, 2)},
    "cli": cli,
}))
shutil.rmtree(wd, ignore_errors=True)
