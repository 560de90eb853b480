"""Device throughput of mashmap-b200-align's hot path (mm_align_batch), one JSON line:
N ONT-like reads (default 100,000 x 10 kb, 2-12 % error; a '-' mapping aligns the same oriented bytes) against their source region of a random
reference (plus 5 % flank on each side), k = (int)((1 - 0.85) * queryLen) as `--pi 85` gives, in batches of --batch reads.
Reports device ms per stage (mm_align_last_stage_ms), aligned Mbp/s (query bases / whole-call time), and the time of the
reference's own edlib call (oracle/_ref/libedlib_ref.so, one CPU thread, as mashmap-align runs it) on the first
--ref-subset pairs when that library is built. Usage: python scripts/align_perf.py [--reads N] [--batch B]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from mashmap_b200 import capi, synth  # noqa: E402


def make_batch(rng, genome, n, read_len):
    qs, ts = [], []
    for _ in range(n):
        flank = read_len // 20
        s = int(rng.integers(flank, len(genome) - read_len - flank))
        src = genome[s : s + read_len]
        q = synth.mutate(src, float(rng.uniform(0.02, 0.12)), rng)
        t = genome[s - flank : s + read_len + flank]
        qs.append(q)
        ts.append(t)
    jobs = np.zeros(n, dtype=capi.align_job_dtype)
    jobs["q_len"] = [len(q) for q in qs]
    jobs["t_len"] = [len(t) for t in ts]
    jobs["q_offset"][1:] = np.cumsum(jobs["q_len"].astype(np.int64))[:-1]
    jobs["t_offset"][1:] = np.cumsum(jobs["t_len"].astype(np.int64))[:-1]
    jobs["k"] = (np.float32(1 - np.float32(85) / np.float32(100)) * jobs["q_len"].astype(np.float32)).astype(np.int32)
    return qs, ts, jobs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=100_000)
    ap.add_argument("--read-len", type=int, default=10_000)
    ap.add_argument("--batch", type=int, default=10_000)
    ap.add_argument("--ref-subset", type=int, default=200)
    a = ap.parse_args()
    rng = np.random.default_rng(11)
    genome = synth.random_genome(1, 50_000_000, seed=12)[0]
    ctx = capi.AlignContext(0)
    stages = np.zeros(8)
    total_ms, qbases, n_aligned = 0.0, 0, 0
    subset = None
    done = 0
    while done < a.reads:
        n = min(a.batch, a.reads - done)
        qs, ts, jobs = make_batch(rng, genome, n, a.read_len)
        if subset is None:
            subset = (qs[: a.ref_subset], ts[: a.ref_subset], jobs[: a.ref_subset].copy())
        res, _ = ctx.align(np.concatenate(qs), np.concatenate(ts), jobs)
        ms = ctx.stage_ms()
        stages[:7] += ms[:7]
        stages[7] = max(stages[7], ms[7])
        total_ms += ms[6]
        qbases += int(jobs["q_len"].sum())
        n_aligned += int((res["alignment_length"] > 0).sum())
        done += n
    ctx.close()
    out = {"workload": f"{a.reads} x {a.read_len} bp reads, 2-12 % error, k from --pi 85, batches of {a.batch}",
           "device_ms": {"h2d": stages[0], "hw_end": stages[1], "shw_start": stages[2], "hirschberg": stages[3],
                         "leaf_traceback": stages[4], "d2h": stages[5], "call_total": stages[6]},
           "max_hirschberg_levels": int(stages[7]), "aligned": n_aligned,
           "aligned_mbp_per_s": qbases / 1e6 / (total_ms / 1e3)}
    try:
        import align_data as AD

        if AD.edlib_ref_available():
            qs, ts, jobs = subset
            t0 = time.perf_counter()
            for q, t, k in zip(qs, ts, jobs["k"]):
                AD.edlib_ref_align(np.ascontiguousarray(q), np.ascontiguousarray(t), int(k))
            dt = time.perf_counter() - t0
            out["reference_edlib"] = {"pairs": len(qs), "s": dt, "ms_per_pair": dt * 1e3 / len(qs),
                                      "mbp_per_s_one_thread": sum(len(q) for q in qs) / 1e6 / dt}
    except Exception as e:  # the reference library is optional
        out["reference_edlib"] = f"not measured: {e}"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
