"""Device index builder on a random reference with one rejected block: how many chunks it re-scans exactly, and how long
the build takes. The block is low-complexity sequence (about two records per position, more than a chunk's record buffer
holds) about 1 Mbp into the first contig.

    python scripts/index_rescan_perf.py [--lib A.so --lib B.so ...] [--reps 3] [--ref-bp 100000000] [--contigs 4]

Each --lib is a build of libmashmap_b200.so (default: the package's own). The builds are run alternately, each in a
process of its own, --reps times; every run prints one JSON line and the card's name and power limit come first."""
import argparse, json, os, subprocess, sys, time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def one_run(lib, ref_bp, contigs, block_at, block_len):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    from mashmap_b200 import capi, synth_gpu

    capi.LIB_PATH = lib
    dev = torch.device("cuda:0")
    ref = synth_gpu.random_reference(contigs, ref_bp // contigs, seed=1, device=dev)
    low = b"ACACACACACGTGTGTGTGT" * (block_len // 20)
    ref[0, block_at : block_at + len(low)] = torch.frombuffer(bytearray(low), dtype=torch.uint8).to(dev)
    torch.cuda.synchronize()
    offs = np.arange(contigs + 1, dtype=np.uint64) * np.uint64(ref_bp // contigs)
    ctx = capi.Context(kmer_size=19, seg_length=5000, sketch_size=220)
    ctx.index_build(None, offs, device_ptr=ref.data_ptr())  # warm-up: module load, allocator
    ctx.close()
    ctx = capi.Context(kmer_size=19, seg_length=5000, sketch_size=220)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = ctx.index_build(None, offs, device_ptr=ref.data_ptr())
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    ctx.close()
    print(json.dumps({"lib": lib, "build_s": round(sec, 4), "scan_s": round(st["ms_scan"] / 1e3, 4), "n_chunks": st["n_chunks"],
                      "n_fixed_chunks": st["n_fixed_chunks"], "fix_rounds": st["fix_rounds"], "n_minmers": st["n_minmers"]}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-bp", type=int, default=100_000_000)
    ap.add_argument("--contigs", type=int, default=4)
    ap.add_argument("--block-at", type=int, default=1_000_000)
    ap.add_argument("--block-len", type=int, default=6000)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    libs = a.lib or [os.path.join(ROOT, "mashmap_b200", "libmashmap_b200.so")]
    if a.child:
        one_run(libs[0], a.ref_bp, a.contigs, a.block_at, a.block_len)
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", q.stdout.strip(), flush=True)
    for _ in range(a.reps):
        for lib in libs:
            subprocess.run([sys.executable, __file__, "--child", "--lib", os.path.abspath(lib), "--ref-bp", str(a.ref_bp),
                            "--contigs", str(a.contigs), "--block-at", str(a.block_at), "--block-len", str(a.block_len)],
                           check=True)


if __name__ == "__main__":
    main()
