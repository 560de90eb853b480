"""Cost of the tag text of `mashmap-b200 --align --eqx / --cs`, one JSON line:
  * the CLI: N ONT-like reads (default 20,000 x 10 kb, 2-12 % error, both strands) against a random reference of
    --ref-mbp Mbp (default 100), the workload of scripts/map_align_perf.py, run with --align, --align --eqx and
    --align --eqx --cs. Reports each wall time and the alignment seconds the CLI prints.
  * one batch through the C ABI: --pairs read-like pairs (default 12,000 x 10 kb at 2-12 % error, about the 256 Mi
    bases of one --align batch) through mm_align_batch_tags with flags 0, EQX and EQX | CS. Reports the call's wall
    time, its stages, the formatting kernels' time (mm_align_last_tag_ms) and the bytes of text returned.
The card's name, power limit and maximum SM clock are read in the same call. Writes its FASTA files to a temporary
directory. Usage: python scripts/align_tags_perf.py [--reads N] [--ref-mbp M] [--pairs P]"""
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
    m = re.search(r"\] (\d+) mappings aligned \(edlib NW over (\d+) query \+ target bases\) in ([0-9.e+-]+) s", p.stderr)
    return dict(wall_s=round(wall, 3), align_s=round(float(m.group(3)), 3), mappings_aligned=int(m.group(1)))


def abi_batch(n_pairs, read_len, seed=7):
    rng = np.random.default_rng(seed)
    ts = [synth.random_genome(1, read_len, seed=seed + 1 + i)[0] for i in range(min(n_pairs, 64))]
    pairs = []
    for i in range(n_pairs):
        t = ts[i % len(ts)]
        pairs.append((synth.mutate(t, float(rng.uniform(0.02, 0.12)), rng), t))
    qb, tb = np.concatenate([p[0] for p in pairs]), np.concatenate([p[1] for p in pairs])
    jobs = np.zeros(n_pairs, dtype=capi.align_job_dtype)
    jobs["q_len"] = [len(p[0]) for p in pairs]
    jobs["t_len"] = [len(p[1]) for p in pairs]
    jobs["q_offset"][1:] = np.cumsum(jobs["q_len"].astype(np.int64))[:-1]
    jobs["t_offset"][1:] = np.cumsum(jobs["t_len"].astype(np.int64))[:-1]
    jobs["k"], jobs["mode"] = -1, capi.MM_ALIGN_NW
    ctx = capi.AlignContext(0, 2 << 30)  # the scratch budget mashmap-b200 --align gives its contexts
    ctx.align_tags(qb[: 2 * read_len], tb[: 2 * read_len], jobs[:1])  # module load, first allocations
    out = dict(pairs=n_pairs, query_plus_target_bases=int(len(qb) + len(tb)))
    for name, flags in (("standard", 0), ("eqx", capi.MM_ALIGN_TAG_EQX),
                        ("eqx_cs", capi.MM_ALIGN_TAG_EQX | capi.MM_ALIGN_TAG_CS)):
        t0 = time.perf_counter()
        res, text = ctx.align_tags(qb, tb, jobs, flags)
        wall = time.perf_counter() - t0
        ms = ctx.stage_ms()
        out[name] = dict(seconds=round(wall, 3), alignment_ops=int(res["alignment_length"].astype(np.int64).sum()),
                         text_bytes=len(text), format_kernels_ms=round(ctx.tag_ms(), 2),
                         stage_ms=dict(h2d=ms[0], distance=ms[1], hirschberg=ms[3], leaves=ms[4], d2h=ms[5]))
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=20_000)
    ap.add_argument("--read-len", type=int, default=10_000)
    ap.add_argument("--ref-mbp", type=int, default=100)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--pairs", type=int, default=12_000)
    a = ap.parse_args()
    out = dict(gpu=gpu_info())
    with tempfile.TemporaryDirectory() as d:
        n_ctg = max(1, a.ref_mbp // 25)
        genome = synth.random_genome(n_ctg, a.ref_mbp * 1_000_000 // n_ctg, seed=101)
        reads, _ = synth.simulate_reads(genome, a.reads, a.read_len, 0.02, 0.12, seed=102)
        ref, qry = os.path.join(d, "ref.fa"), os.path.join(d, "reads.fa")
        synth.write_fasta(ref, [f"ctg{i}" for i in range(n_ctg)], genome)
        synth.write_fasta(qry, [f"read{i}" for i in range(len(reads))], reads)
        base = ["-r", ref, "-q", qry, "--pi", "85", "-t", str(a.threads), "--align"]
        run_cli(base + ["-o", os.path.join(d, "warm.paf")])  # first device use of the run: module load, allocations
        cli = dict(reference_bp=sum(len(c) for c in genome), reads=len(reads), read_len=a.read_len, threads=a.threads)
        for name, extra in (("align", []), ("align_eqx", ["--eqx"]), ("align_eqx_cs", ["--eqx", "--cs"])):
            cli[name] = run_cli(base + extra + ["-o", os.path.join(d, f"{name}.paf")])
        out["cli"] = cli
    out["abi_batch"] = abi_batch(a.pairs, a.read_len)
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
