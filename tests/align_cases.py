"""End-to-end cases of mashmap-b200-align (tests/test_gpu_align.py, tests/golden/make_align_golden.py): deterministic
inputs written to a directory, the mapping file each case aligns, and the command-line options. Mapping files made by a
mapper are stored under tests/golden/align/ (the mapper is checked against them separately); hand-made ones are written
here."""
from __future__ import annotations

import os

import numpy as np

from mashmap_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "align")


def write_inputs(d):
    """genome (2 x 150 kb), 40 ONT-like 10 kb reads at 2-14 % error on both strands (every 8th with an N run) split over
    two files, and one 250 kb read for a mapping that needs several Hirschberg levels"""
    os.makedirs(d, exist_ok=True)
    genome = synth.random_genome(2, 150_000, seed=31)
    gnames = ["chrA", "chrB"]
    reads, _ = synth.simulate_reads(genome, 40, 10_000, 0.02, 0.14, seed=32)
    for i in range(0, len(reads), 8):
        reads[i] = reads[i].copy()
        reads[i][3000:3150] = ord("N")
    names = [f"read{i}" for i in range(len(reads))]
    synth.write_fasta(os.path.join(d, "ref.fa"), gnames, genome)
    synth.write_fasta(os.path.join(d, "reads.fa"), names, reads)
    synth.write_fasta(os.path.join(d, "reads1.fa"), names[:20], reads[:20])
    synth.write_fasta(os.path.join(d, "reads2.fa"), names[20:], reads[20:])
    with open(os.path.join(d, "reads.list"), "w") as f:
        f.write(os.path.join(d, "reads1.fa") + "\n" + os.path.join(d, "reads2.fa") + "\n")
    big_ref = synth.random_genome(1, 300_000, seed=33)[0]
    rng = np.random.default_rng(34)
    big = synth.mutate(big_ref[20_000:270_000], 0.05, rng)
    synth.write_fasta(os.path.join(d, "bigref.fa"), ["big"], [big_ref])
    synth.write_fasta(os.path.join(d, "bigread.fa"), ["bigread"], [big])
    with open(os.path.join(d, "big.map"), "w") as f:
        f.write(f"bigread {len(big)} 0 {len(big) - 1} + big 300000 20000 269999 95.0\n")
    # hand-made v3-style lines (exclusive ends): an end equal to the sequence length takes in its terminating NUL, on the
    # query side, the target side or both, on both strands
    tail = synth.mutate(genome[0][-6000:], 0.05, rng)
    tail_r = synth.revcomp(tail)
    synth.write_fasta(os.path.join(d, "nulreads.fa"), ["tailF", "tailR"], [tail, tail_r])
    n = len(tail)
    lines = [
        f"tailF {n} 1 {n} + chrA 150000 144000 150000 90.0",
        f"tailF {n} 0 {n - 1} + chrA 150000 144001 150000 90.0",
        f"tailF {n} 2 {n} + chrA 150000 144000 149999 90.0",
        f"tailR {n} 1 {n} - chrA 150000 144000 150000 90.0",
        f"tailR {n} 0 {n - 1} - chrA 150000 144001 150000 90.0",
    ]
    with open(os.path.join(d, "nul.map"), "w") as f:
        f.write("\n".join(lines) + "\n")
    return d


MAPPED = os.path.join(GOLDEN, "reads_legacy.map")  # `mashmap --legacy -r ref.fa -q reads.fa --pi 80`

# name -> (subject, query option, query, mapping file, extra options)
CASES = {
    "ont_pi90": ("ref.fa", "-q", "reads.fa", MAPPED, ["--pi", "90"]),
    "ont_pi80": ("ref.fa", "-q", "reads.fa", MAPPED, ["--pi", "80"]),
    "ont_pi0": ("ref.fa", "-q", "reads.fa", MAPPED, ["--pi", "0"]),
    "ont_querylist": ("ref.fa", "--ql", "reads.list", MAPPED, ["--pi", "85"]),
    "nul_v3": ("ref.fa", "-q", "nulreads.fa", "nul.map", ["--pi", "70"]),
    "long_250kb": ("bigref.fa", "-q", "bigread.fa", "big.map", ["--pi", "85"]),
}


def case_args(d, name):
    subj, qopt, query, mapping, extra = CASES[name]
    mp = mapping if os.path.isabs(mapping) else os.path.join(d, mapping)
    return ["-s", os.path.join(d, subj), qopt, os.path.join(d, query), "--mappingFile", mp] + extra
