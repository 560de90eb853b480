"""Cost of long alignments (the banded CTA path of mm_align.cu), one JSON line:
  * single MM_ALIGN_NW pairs (default 100 kb, 1 Mbp and 5 Mbp at 1 % and 5 %, the query a synth.mutate copy of the
    target): the mm_align_batch call's wall time, its stages (mm_align_last_stage_ms) and the number of Hirschberg
    levels; with the unmodified edlib's one-thread CPU time on the same pair where oracle/_ref is built (pairs up to
    --edlib-max-bp, default 1 Mbp).
  * the routing rule: NW pairs of MM_ALIGN_BAND_MIN_LEN - 1 (warp path) and MM_ALIGN_BAND_MIN_LEN (banded) bases.
  * throughput: one batch of --batch (default 200) 1 Mbp pairs at 1 %.
  * the assembly-like CLI case of tests/test_gpu_align_band.py (1.2 + 2.5 + 4 Mbp, -s 10000 --pi 95): wall time
    without and with --align --alignMaxLen 5000000, in the default mode and with -f one-to-one.
The card's name, power limit and maximum SM clock are read in the same run. Writes its files to a temporary directory.
Usage: python scripts/align_band_perf.py [--batch N]"""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mashmap_b200 import capi, synth  # noqa: E402

MAP_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200")
EDLIB = os.path.join(ROOT, "oracle", "_ref", "libedlib_nw_ref.so")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def pair(n, div, seed):
    rng = np.random.default_rng(seed)
    t = synth.random_sequence(n, rng)
    return np.ascontiguousarray(synth.mutate(t, div, rng)), t


def batch_jobs(pairs):
    jobs = np.zeros(len(pairs), dtype=capi.align_job_dtype)
    jobs["q_len"] = [len(p[0]) for p in pairs]
    jobs["t_len"] = [len(p[1]) for p in pairs]
    jobs["q_offset"][1:] = np.cumsum(jobs["q_len"].astype(np.int64))[:-1]
    jobs["t_offset"][1:] = np.cumsum(jobs["t_len"].astype(np.int64))[:-1]
    jobs["k"], jobs["mode"] = -1, capi.MM_ALIGN_NW
    return np.concatenate([p[0] for p in pairs]), np.concatenate([p[1] for p in pairs]), jobs


def device_call(ctx, pairs):
    qb, tb, jobs = batch_jobs(pairs)
    t0 = time.perf_counter()
    res, _ = ctx.align(qb, tb, jobs)
    wall = time.perf_counter() - t0
    ms = ctx.stage_ms()
    return res, wall, dict(h2d=round(ms[0], 2), distance=round(ms[1], 2), hirschberg=round(ms[3], 2),
                           leaves=round(ms[4], 2), d2h=round(ms[5], 2), hirschberg_levels=int(ms[7]))


def edlib_seconds(q, t):
    import align_nw_data as AN

    t0 = time.perf_counter()
    ed = AN.edlib_ref_align_nw(q, t, -1)[0]
    return ed, time.perf_counter() - t0


def run_cli(args):
    t0 = time.perf_counter()
    p = subprocess.run([MAP_BIN] + args, capture_output=True, text=True)
    if p.returncode != 0:
        raise RuntimeError(p.stderr[-3000:])
    return time.perf_counter() - t0, p.stderr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000, 5_000_000])
    ap.add_argument("--divs", type=float, nargs="+", default=[0.01, 0.05])
    ap.add_argument("--edlib-max-bp", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=200)
    a = ap.parse_args()
    out = dict(gpu=gpu_info(), band_min_len=capi.MM_ALIGN_BAND_MIN_LEN)
    ctx = capi.AlignContext(0, 2 << 30)  # the scratch budget mashmap-b200 --align gives its contexts
    device_call(ctx, [pair(1000, 0.01, 1)])  # module load, first allocations
    singles = []
    for n in a.sizes:
        for div in a.divs:
            q, t = pair(n, div, 11)
            res, wall, st = device_call(ctx, [(q, t)])
            row = dict(bp=n, divergence=div, ed=int(res[0]["ed"]), seconds=round(wall, 3), stage_ms=st)
            if os.path.exists(EDLIB) and n <= a.edlib_max_bp:
                ed, sec = edlib_seconds(q, t)
                row.update(edlib_cpu_1thread_s=round(sec, 3), edlib_ed=int(ed), speedup=round(sec / wall, 2))
            singles.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    out["single_pairs"] = singles
    rule = []
    L = capi.MM_ALIGN_BAND_MIN_LEN
    for div in (0.01, 0.05):
        for n, path in ((L - 1, "warp"), (L, "band")):
            ps = [pair(n, div, 20 + i) for i in range(8)]
            _, wall, st = device_call(ctx, ps)
            rule.append(dict(bp=n, divergence=div, path=path, jobs=len(ps), seconds=round(wall, 4), stage_ms=st))
    out["routing_rule"] = rule
    ps = [pair(1_000_000, 0.01, 100 + i) for i in range(a.batch)]
    res, wall, st = device_call(ctx, ps)
    bases = sum(len(p[0]) + len(p[1]) for p in ps)
    out["batch_1mbp"] = dict(jobs=len(ps), divergence=0.01, seconds=round(wall, 3), stage_ms=st,
                             pairs_per_s=round(len(ps) / wall, 2), query_plus_target_mbp_per_s=round(bases / wall / 1e6, 1),
                             all_aligned=bool((res["ed"] >= 0).all() and (res["alignment_length"] > 0).all()))
    ctx.close()
    import align_band_data as AB

    with tempfile.TemporaryDirectory() as d:
        ref, qry = AB.write_asm(d)
        cli = {}
        base = ["-r", ref, "-q", qry] + AB.ASM_OPTS
        run_cli(base + ["-o", os.path.join(d, "warm.paf")])
        for mode, opts in sorted(AB.ASM_MODES.items()):
            w0, _ = run_cli(base + opts + ["-o", os.path.join(d, "plain.paf")])
            w1, err = run_cli(base + opts + ["-o", os.path.join(d, "align.paf"), "--align", "--alignMaxLen", "5000000"])
            m = re.search(r"\] (\d+) mappings aligned \(edlib NW over (\d+) query \+ target bases\) in ([0-9.e+-]+) s", err)
            lens = [max(int(f[3]) - int(f[2]), int(f[8]) - int(f[7]))
                    for f in (ln.split("\t") for ln in open(os.path.join(d, "align.paf")))]
            cli[mode] = dict(wall_s_without_align=round(w0, 3), wall_s_with_align=round(w1, 3),
                             align_s=float(m.group(3)) if m else None, mappings=len(lens), longest_mapping_bp=max(lens))
        out["assembly_cli"] = cli
    print(json.dumps(out))


if __name__ == "__main__":
    main()
