"""Awkward FASTQ files for the FASTQ window reader's tests: every case where the four-lines-per-record rule of the line
reader (skch_seqio.cpp, for_each_seq_in_file) is easy to get wrong."""
from __future__ import annotations

import numpy as np

IUPAC = b"ACGTacgtNnRYKMSWBDHVryk"


def dna(rng, n, alphabet=b"ACGT"):
    return np.frombuffer(alphabet, dtype=np.uint8)[rng.integers(0, len(alphabet), n)].tobytes()


def fastq(rng, n_rec, lens, header=b"@r%d desc", alphabet=b"ACGT", qual_first=b"I"):
    out = []
    for i in range(n_rec):
        s = dna(rng, int(rng.choice(lens)), alphabet)
        q = (qual_first + b"I" * len(s))[: len(s)]
        out.append((header % i if b"%d" in header else header) + b"\n" + s + b"\n+\n" + q + b"\n")
    return b"".join(out)


def awkward(seed=0):
    """{name: text}; "empty_header" is the one case the reference's own reader throws on"""
    rng = np.random.default_rng(seed)
    base = fastq(rng, 40, [0, 1, 2, 59, 60, 61, 700])
    return {
        "plain": base,
        "crlf": base.replace(b"\n", b"\r\n"),
        "no_final_newline": base.rstrip(b"\n"),
        "cut_after_1": base + b"@tail one",
        "cut_after_1_nl": base + b"@tail one\n",
        "cut_after_2": base + b"@tail two\nACGTA",
        "cut_after_2_nl": base + b"@tail two\nACGTA\n",
        "cut_after_3": base + b"@tail three\nACGTAC\n+",
        "cut_after_3_nl": base + b"@tail three\nACGTAC\n+\n",
        "empty_header": fastq(rng, 10, [5, 70]) + b"\n" + fastq(rng, 5, [30]),
        "empty_header_at_end": base + b"\n",
        "headers": b"@noSpace\nACGT\n+\nIIII\n@tab\there x\nAC\n+\nII\n@ leading space here\nACG\n+\nIII\n@\nA\n+\nI\n"
                   b"@two  spaces\nTT\n+\nII\n space first x\nCA\n+\nII\nno at sign\nGA\n+\nII\n@cr\r\nGG\r\n+\r\nII\r\n",
        "quality_at_plus": fastq(rng, 30, [1, 5, 80], qual_first=b"@") + fastq(rng, 30, [1, 5, 80], qual_first=b"+"),
        "empty_sequences": fastq(rng, 20, [0]) + fastq(rng, 20, [0, 3]),
        "iupac_lowercase": fastq(rng, 50, [1, 2, 3, 31, 32, 33, 999], alphabet=IUPAC),
        "odd_lengths": fastq(rng, 60, [1, 3, 5, 7, 63, 65, 1001]),
        "long_record": fastq(rng, 2, [50]) + fastq(rng, 1, [300_000], header=b"@long") + fastq(rng, 3, [10]),
    }
