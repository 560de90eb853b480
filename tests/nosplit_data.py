"""Inputs of the tests of queries mapped as ONE fragment longer than a segment (--noSplit, windowLen > 0), and the
reference's stored results for them (tests/golden/nosplit_digests.json and tests/golden/nosplit/*.paf, written by
tests/golden/make_nosplit_golden.py from the unmodified reference)."""
from __future__ import annotations

import json
import os

import numpy as np

from mashmap_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "golden", "nosplit_digests.json")
PAF_DIR = os.path.join(HERE, "golden", "nosplit")

SEG = 5000
# (k, s) of the sketch tests: the smallest, the default and the largest k-mer size
SKETCH_CASES = [(8, 50), (19, 100), (32, 200)]

_store = None


def long_sequences(k, seg=SEG):
    """Fragments of seg+1, 2*seg, 10*seg+r and >= 1 Mbp bases, N runs across the boundaries of the pieces the device cuts
    a long fragment into (piece j starts at j*(seg-k+1)), homopolymers, tandem repeats (fewer than s distinct k-mers),
    palindromes (vote sums of 0), all-N, and repeats whose copies fall into different pieces."""
    rng = np.random.default_rng(1000 + k)
    step = seg - k + 1
    N = ord("N")
    out = [synth.random_sequence(seg + 1, rng)]
    b = synth.random_sequence(2 * seg, rng)
    b[step - 3 : step + 3] = N
    out.append(b)
    c = synth.random_sequence(10 * seg + 137, rng)
    c[0] = N
    for j in (1, 2, 5, 9):
        c[j * step - 2 : j * step + k] = N  # a run that ends exactly where a k-mer of the next piece would start
    c[3 * step + 1 : 3 * step + 2] = N
    c[-3:] = N
    out.append(c)
    d = synth.random_sequence(1_000_003, rng)
    for j in range(7, 200, 31):
        d[j * step - k // 2 : j * step + k // 2] = N
    out.append(d)
    out.append(np.full(3 * seg + 5, ord("A"), np.uint8))
    out.append(np.tile(np.frombuffer(b"ACGTTGCAAG", np.uint8), (4 * seg + 7) // 10 + 1)[: 4 * seg + 7])
    out.append(np.tile(synth.random_sequence(300, rng), 6 * seg // 300 + 1)[: 6 * seg])
    pal = synth.random_sequence(seg + 1, rng)
    out.append(np.concatenate([pal, synth.revcomp(pal)]))
    out.append(np.full(2 * seg, N, np.uint8))
    unit = synth.random_sequence(2 * seg + 11, rng)
    out.append(np.concatenate([unit, synth.random_sequence(700, rng), unit, unit]))  # the same k-mers in several pieces
    out.append(np.frombuffer(b"acgtnACGTRYKM" * (3 * seg // 13), np.uint8).copy())
    return out


def short_sequences():
    """ordinary segments that share a batch with the long fragments"""
    rng = np.random.default_rng(77)
    return [synth.random_sequence(SEG, rng), synth.random_sequence(57, rng), synth.random_sequence(SEG - 1, rng),
            np.full(SEG, ord("C"), np.uint8)]


def load():
    global _store
    if _store is None:
        _store = json.load(open(PATH)) if os.path.exists(PATH) else {}
    return _store


def get(section, key):
    v = load().get(section, {}).get(key)
    assert v is not None, f"no stored reference result for {section} / {key}: run tests/golden/make_nosplit_golden.py"
    return v


def check_stored(section, key, value):
    """with the reference built: the stored digests must still be what the reference computes"""
    stored = load().get(section, {}).get(key)
    if stored is not None:
        assert stored == value, f"tests/golden/nosplit_digests.json is stale for {section} / {key}"


# Stage parity of whole queries mapped as one fragment (test_gpu_nosplit.py): data set and command line (the sessions the
# stage tests of tests/test_gpu_stages.py use, whose parameters / index / tables are stored in reference_digests.json)
STAGE_RUNS = [("random", ["-s", "5000", "--pi", "85", "-t", "4"]), ("panel", ["-s", "5000", "--pi", "85", "-t", "4"]),
              ("asm", ["-s", "10000", "--pi", "90", "-f", "one-to-one", "-t", "4"]), ("rep", ["-s", "5000", "--pi", "85", "-t", "4"]),
              ("rep", ["-s", "5000", "--pi", "85", "--noHgFilter", "-t", "4"])]

# mashmap-b200 --noSplit against the reference CLI (test_gpu_nosplit.py); the reference's PAF is stored as
# tests/golden/nosplit/<cli_name(...)>.paf
CLI_RUNS = [("random", ["-s", "5000", "--pi", "85"]), ("random", ["-s", "5000", "--pi", "95", "--dense", "-f", "none"]),
            ("panel", ["-s", "5000", "--pi", "85"]), ("panel", ["-s", "5000", "--pi", "95", "-n", "2", "-Y", "#"]),
            ("panel", ["-s", "3000", "--pi", "90", "-f", "one-to-one", "-X"]),
            ("panel", ["-s", "5000", "--pi", "90", "--lowerTriangular", "-n", "2"]),
            ("assembly", ["-s", "10000", "--pi", "90", "-f", "one-to-one"]), ("repeat", ["-s", "5000", "--pi", "85"]),
            ("repeat", ["-s", "5000", "--pi", "85", "--noHgFilter", "-f", "map", "-n", "2"])]


def datasets_by_name(workdir):
    import datasets

    return {"random": lambda: datasets.make_random_set(workdir), "panel": lambda: datasets.make_panel_set(workdir),
            "asm": lambda: datasets.make_assembly_set(workdir), "assembly": lambda: datasets.make_assembly_set(workdir),
            "rep": lambda: datasets.make_repeat_set(workdir), "repeat": lambda: datasets.make_repeat_set(workdir)}


def cli_name(which, args):
    return which + "_" + "_".join(a.strip("-#").replace("#", "hash") or "hash" for a in args)


def whole_reads(d, k):
    """every query of the data set as ONE fragment (what skch::Map does under --noSplit): (read index, length) of the reads
    with at least k bases"""
    idx = [i for i, r in enumerate(d["reads"]) if len(r) >= k]
    return np.array(idx, dtype=np.int64), np.array([len(d["reads"][i]) for i in idx], dtype=np.int64)
