"""Cost of `mashmap-b200 --align`, one JSON line:
  * mapping against alignment: N ONT-like reads (default 20,000 x 10 kb, 2-12 % error, both strands) against a random
    reference of --ref-mbp Mbp (default 100), mapped by the CLI once without and once with --align (--pi 85, -t
    --threads). Reports both wall times, the alignment seconds the CLI prints, and the aligned rate in query bases and in
    query + target bases per second.
  * one long alignment: a --long-bp x --long-bp pair (default 1 Mbp, the query a 5 % diverged copy of the target) through
    mm_align_batch with MM_ALIGN_NW, as --align sends a 1 Mbp one-to-one mapping; reports the call's wall time and its
    stages (mm_align_last_stage_ms). This time is what --alignMaxLen's default is set from.
Writes its FASTA files to a temporary directory. Usage: python scripts/map_align_perf.py [--reads N] [--ref-mbp M]"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from mashmap_b200 import capi, synth  # noqa: E402

MAP_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def run_cli(args):
    t0 = time.perf_counter()
    p = subprocess.run([MAP_BIN] + args, capture_output=True, text=True)
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        raise RuntimeError(p.stderr[-3000:])
    return wall, p.stderr


def long_alignment(n, seed=9):
    rng = np.random.default_rng(seed)
    t = synth.random_genome(1, n, seed=seed)[0]
    q = synth.mutate(t, 0.05, rng)[:n]
    jobs = np.zeros(1, dtype=capi.align_job_dtype)
    jobs["q_len"], jobs["t_len"], jobs["k"], jobs["mode"] = len(q), len(t), -1, capi.MM_ALIGN_NW
    ctx = capi.AlignContext(0, 2 << 30)  # the scratch budget mashmap-b200 --align gives its contexts
    t0 = time.perf_counter()
    res, ops = ctx.align(q, t, jobs)
    wall = time.perf_counter() - t0
    ms = ctx.stage_ms()
    ctx.close()
    return dict(q_len=int(len(q)), t_len=int(len(t)), ed=int(res[0]["ed"]), seconds=round(wall, 3),
                stage_ms=dict(h2d=ms[0], distance=ms[1], hirschberg=ms[3], leaves=ms[4], d2h=ms[5]),
                hirschberg_levels=int(ms[7]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000)
    ap.add_argument("--read-len", type=int, default=10_000)
    ap.add_argument("--ref-mbp", type=int, default=100)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--long-bp", type=int, nargs="+", default=[100_000, 1_000_000])
    a = ap.parse_args()
    out = dict(gpu=gpu_info())
    with tempfile.TemporaryDirectory() as d:
        n_ctg = max(1, a.ref_mbp // 25)
        genome = synth.random_genome(n_ctg, a.ref_mbp * 1_000_000 // n_ctg, seed=101)
        reads, _ = synth.simulate_reads(genome, a.reads, a.read_len, 0.02, 0.12, seed=102)
        ref, qry = os.path.join(d, "ref.fa"), os.path.join(d, "reads.fa")
        synth.write_fasta(ref, [f"ctg{i}" for i in range(n_ctg)], genome)
        synth.write_fasta(qry, [f"read{i}" for i in range(len(reads))], reads)
        base = ["-r", ref, "-q", qry, "--pi", "85", "-t", str(a.threads)]
        run_cli(base + ["-o", os.path.join(d, "warm.paf")])  # first device use of the run: module load, allocations
        w_map, _ = run_cli(base + ["-o", os.path.join(d, "plain.paf")])
        w_aln, err = run_cli(base + ["-o", os.path.join(d, "align.paf"), "--align"])
        m = re.search(r"\] (\d+) mappings aligned \(edlib NW over (\d+) query \+ target bases\) in ([0-9.e+-]+) s", err)
        n_aln, bases, sec = int(m.group(1)), int(m.group(2)), float(m.group(3))
        qbases = 0
        for line in open(os.path.join(d, "align.paf")):
            f = line.split("\t")
            if "\tcg:Z:" in line:
                qbases += int(f[3]) - int(f[2])
        out["map_vs_align"] = dict(
            reference_bp=sum(len(c) for c in genome), reads=len(reads), read_len=a.read_len, threads=a.threads,
            wall_s_without_align=round(w_map, 3), wall_s_with_align=round(w_aln, 3), align_s=round(sec, 3),
            mappings_aligned=n_aln, aligned_query_mbp_per_s=round(qbases / sec / 1e6, 2),
            aligned_query_plus_target_mbp_per_s=round(bases / sec / 1e6, 2))
    out["long_alignment"] = [long_alignment(n) for n in a.long_bp]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
