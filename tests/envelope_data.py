"""Inputs of the tests at the edges of the mapping kernels' parameter envelope (tests/test_gpu_envelope.py,
tests/test_envelope_cpu.py): segment lengths from the reference's minimum (100) to 50 kb, sketch sizes from 1 to the
largest a context accepts, the sizes where a kernel changes its code path, k-mer sizes the full pipeline is not run at
elsewhere. The reference's results for them are stored in tests/golden/reference_digests.json (sections "sessions" and
"fragments") and tests/golden/envelope/*.paf, written by tests/golden/make_envelope_golden.py."""
from __future__ import annotations

import os

import numpy as np

from mashmap_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
PAF_DIR = os.path.join(HERE, "golden", "envelope")


def make_envelope_sets(workdir, tag="env", seed=81):
    """One 1.2 Mbp random reference and three query files against it, each with reads shorter than a segment and ragged
    last fragments:
      reads  30 noisy 10 kb reads, 10 of 80-400 bp, 12,345 bp with an N run, 3,217 bp lower case with IUPAC codes
      short  40 reads of 80-400 bp, three 10 kb reads, 1,234 bp (segments of 100 bp)
      long   four 120 kb reads, 57,123 bp, 23,456 bp, two 10 kb reads, 3,000 bp (segments of 20 and 50 kb)
    Returns {name: data set} in the layout of tests/datasets.py."""
    genome = synth.random_genome(3, 400_000, seed=seed)
    names = [f"ctg{i}" for i in range(len(genome))]
    ref = os.path.join(workdir, f"{tag}_ref.fa")
    synth.write_fasta(ref, names, genome)
    rng = np.random.default_rng(seed + 1)

    def short_reads(n, s):
        lens = rng.integers(80, 401, n)
        return [synth.simulate_reads(genome, 1, int(x), 0.0, 0.05, seed=s + i)[0][0] for i, x in enumerate(lens)]

    def noisy(n, length, lo, hi, s):
        return synth.simulate_reads(genome, n, length, lo, hi, seed=s)[0]

    odd = genome[1][50_000:62_345].copy()
    odd[3000:3400] = ord("N")
    low = np.frombuffer(genome[2][10_000:13_217].tobytes().lower(), dtype=np.uint8).copy()
    low[::97] = ord("R")
    queries = {
        "reads": noisy(30, 10_000, 0.01, 0.10, seed + 10) + short_reads(10, seed + 100) + [odd, low],
        "short": short_reads(40, seed + 200) + noisy(3, 10_000, 0.01, 0.05, seed + 20) + noisy(1, 1_234, 0.01, 0.03, seed + 21),
        "long": (noisy(4, 120_000, 0.002, 0.01, seed + 30) + noisy(1, 57_123, 0.005, 0.02, seed + 31)
                 + noisy(1, 23_456, 0.005, 0.02, seed + 32) + noisy(2, 10_000, 0.01, 0.05, seed + 33)
                 + noisy(1, 3_000, 0.01, 0.03, seed + 34)),
    }
    out = {}
    for name, reads in queries.items():
        qry = os.path.join(workdir, f"{tag}_{name}.fa")
        rnames = [f"{name}{i}" for i in range(len(reads))]
        synth.write_fasta(qry, rnames, reads)
        synth.write_fai(qry, rnames, reads)
        out[name] = dict(ref=ref, qry=qry, genome=genome, names=names, reads=reads, rnames=rnames)
    return out


def make_locus_slot_sets(workdir):
    """tests/datasets.py's repeat set with a tandem array of 2 and of 3 copies: one L1 candidate over the array gives
    exactly as many equally good loci"""
    import datasets

    return {f"tandem{n}": datasets.make_repeat_set(workdir, tag=f"envrep{n}", tandem_copies=n) for n in (2, 3)}


def largest_sketch_size(seg_length, kmer_size=19):
    """the largest sketch size mm_params_check accepts at this segment length"""
    from mashmap_b200 import capi

    s = 1
    while capi.params_check(kmer_size, seg_length, s + 1)[0] == 0:
        s += 1
    return s


def stage_runs():
    """(row, data set, options, diag counters that prove the row's path ran with the fast kernels) of every stage-parity
    row"""
    runs = []
    for j in (1, 2, 3):  # K1's threshold constant, k_l2_prep's first-level table and the cut-off table at s = 1..3
        runs.append(("tiny sketch", "reads", ["-s", "1000", "-J", str(j)], ()))
    for s in (100, 101):  # the reference's shortest segment: ~82 k-mer positions, K1's list capacities at their clamps
        runs.append(("shortest segments", "short", ["-s", str(s), "--pi", "85"], ()))
    for j in (256, 257):  # k_l1_warp's hit list in the scan arrays' space / in its own region
        runs.append(("hit-list aliasing", "reads", ["-s", "5000", "-J", str(j)], ()))
    # From s = 900 on, the hypergeometric cut-off table depends on how the GSL stand-in the reference is built with
    # (oracle/gsl_shim) sums its terms: the stand-in of earlier oracle builds moves entries by up to 4 there, against the
    # exact values the product computes (tests/test_envelope_cpu.py). The K3 switches below do not depend on that table,
    # so these rows run without the hypergeometric filter and compare the same with any build of the stand-in.
    no_hg = ["--noHgFilter"]
    for j in (1000, 1001):  # the last sketch size of k_l2_scan's 11-bit counters / the first all-k_l2 size
        runs.append(("stream limit", "reads", ["-s", "5000", "-J", str(j)] + no_hg, ()))
    runs.append(("reference's rule", "reads", ["-s", "10000", "--dense", "--pi", "80"] + no_hg, ()))  # s = 998
    runs.append(("reference's rule", "long", ["-s", "20000", "--dense", "--pi", "85"] + no_hg, ()))  # s = 1598
    for seg, which in ((5000, "reads"), (20000, "long")):  # k_l2 at its shared-memory / live-set limit
        runs.append(("general L2 limit", which, ["-s", str(seg), "-J", str(largest_sketch_size(seg))] + no_hg, ()))
    for seg in (20000, 50000):  # K1's list capacity lowered until its layout fits
        runs.append(("long segments", "long", ["-s", str(seg)], ()))
    runs.append(("locus slots", "tandem2", ["-s", "5000", "--pi", "85", "--noHgFilter"], ()))
    runs.append(("locus slots", "tandem3", ["-s", "5000", "--pi", "85", "--noHgFilter"], ("l2_general_cands",)))
    for k in (8, 12, 24, 28):  # K2 / K3 at k-mer sizes the full pipeline is not run at elsewhere
        runs.append(("k-mer size", "reads", ["-s", "5000", "-k", str(k)], ()))
    return [(row, which, opts + ["-t", "4"], diag) for row, which, opts, diag in runs]


# mashmap-b200 against the reference CLI; the reference's PAF is stored as tests/golden/envelope/<cli_name(...)>.paf
CLI_RUNS = [("short", ["-s", "100", "--pi", "85"]), ("reads", ["-s", "1000", "-J", "1"]),
            ("reads", ["-s", "5000", "-J", "1001"]), ("long", ["-s", "20000", "--dense", "--pi", "85"])]


def cli_name(which, args):
    return which + "_" + "_".join(a.strip("-") for a in args)


def datasets_by_name(workdir):
    sets = {}

    def get(name):
        if name not in sets:
            sets.update(make_locus_slot_sets(workdir) if name.startswith("tandem") else make_envelope_sets(workdir))
        return sets[name]

    return get
