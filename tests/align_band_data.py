"""Cases of the banded long-alignment path (tests/test_gpu_align_band.py) and their checker: the unmodified edlib
(oracle/_ref/libedlib_nw_ref.so for NW, libedlib_ref.so for HW) where it is built, otherwise the sha256 digests of its
results stored in tests/golden/align_band/ by tests/golden/make_align_band_golden.py. Test infrastructure only."""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np

import align_data as AD
import align_nw_data as AN
from mashmap_b200 import capi, synth

GOLDEN = os.path.join(AD.ROOT, "tests", "golden", "align_band", "edlib_digests.json")
L = capi.MM_ALIGN_BAND_MIN_LEN


def key(q, t, k, mode):
    h = hashlib.sha256()
    for a in (q, t):
        h.update(hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).digest())
    h.update(f"{int(k)},{int(mode)}".encode())
    return h.hexdigest()


def digest(ed, start, end, ops):
    return hashlib.sha256(f"{ed},{start},{end},".encode() + np.asarray(ops, dtype=np.uint8).tobytes()).hexdigest()


def edlib_available():
    return AN.edlib_nw_ref_available() and AD.edlib_ref_available()


def edlib(q, t, k, mode):
    """(ed, start, end, ops) of the unmodified edlib"""
    f = AN.edlib_ref_align_nw if mode == capi.MM_ALIGN_NW else AD.edlib_ref_align
    return f(q, t, k)[:4]


def cigar_digest(cigar):
    return hashlib.sha256(cigar.encode()).hexdigest()


def golden_entry(q, t, k, mode):
    """[ed, digest of (ed, start, end, ops), digest of the standard CIGAR] from the unmodified edlib"""
    r = edlib(q, t, k, mode)
    return [r[0], digest(*r), cigar_digest(AD.cigar(r[3]))]


_golden = None


def want(q, t, k, mode):
    """[ed, digest of (ed, start, end, ops), digest of the CIGAR] of edlibAlign(mode, PATH): edlib where built, the
    stored digests otherwise"""
    global _golden
    if edlib_available():
        return golden_entry(q, t, k, mode)
    if _golden is None:
        with open(GOLDEN) as f:
            _golden = json.load(f)
    return _golden[key(q, t, k, mode)]


# ---- pairs ----------------------------------------------------------------------------------------------------------

def _features(src, rng):
    """N runs, a homopolymer and a tandem repeat written into a copy of src"""
    s = src.copy()
    n = len(s)
    for _ in range(3):
        a = int(rng.integers(0, n)); s[a : a + int(rng.integers(1, 300))] = ord("N")
    a = int(rng.integers(0, n)); s[a : a + 400] = ord("A")
    a = int(rng.integers(0, n)); seg = s[a : a + 3000]; s[a : a + len(seg)] = np.resize(AD._ACGT[[0, 2, 3]], len(seg))
    return s


def _indels(q, rng, sizes):
    """long deletions and insertions (sizes) at random places of q"""
    for sz in sizes:
        at = int(rng.integers(0, max(1, len(q) - sz)))
        if rng.random() < 0.5:
            q = np.concatenate([q[:at], q[at + sz :]])
        else:
            q = np.concatenate([q[:at], AD._ACGT[rng.integers(0, 4, size=sz)], q[at:]])
    return q


def nw_pairs():
    """(name, query, target) pairs around and above the routing rule: lengths L - 1, L, L + 1, 2L, 200 kb, 1 Mbp (the
    target's length; the query's differs by the indels), 0-15 % divergence, long indels, N runs, homopolymers, tandem
    repeats, query lengths 0 / 1 / 63 mod 64"""
    rng = np.random.default_rng(2026)
    out = []
    for n in (L - 1, L, L + 1, 2 * L, 200_000, 1_000_000):
        for div in (0.0, 0.001, 0.01, 0.05, 0.15):
            if n == 1_000_000 and div > 0.05:
                continue  # keeps edlib's CPU time for the file to a few minutes
            t = synth.random_sequence(n, rng)
            if n <= 2 * L:
                t = _features(t, rng)
            q = synth.mutate(t, div, rng) if div > 0 else t.copy()
            if div >= 0.01 and n <= 200_000:
                q = _indels(q, rng, (80, 1500))
            out.append((f"nw{n}_{div}", np.ascontiguousarray(q, dtype=np.uint8), t))
    for r in (0, 1, 63):  # query lengths by their last block, a close copy of a target of the rule's length
        t = synth.random_sequence(L, rng)
        q = synth.mutate(t, 0.01, rng)
        m = len(q) // 64 * 64 + r
        q = np.resize(q, m) if m <= len(q) else np.concatenate([q, t[: m - len(q)]])
        out.append((f"mod64_{r}", np.ascontiguousarray(q, dtype=np.uint8), t))
    return out


def k_variants(q, t, ed):
    """the k = -1 case decides ed; these bounds decide the same distance or -1 with edlib's rule"""
    ks = [ed, max(0, ed - 1)]
    d = abs(len(q) - len(t))
    if d > 0:
        ks.append(d - 1)  # below the length difference
    return ks


def hw_pairs():
    """(name, query, target) HW cases whose Hirschberg nodes are long: a query inside a slightly longer target"""
    rng = np.random.default_rng(2027)
    out = []
    for qlen, tlen, div in ((150_000, 160_000, 0.01), (150_000, 160_000, 0.05), (400_000, 420_000, 0.02)):
        t = synth.random_sequence(tlen, rng)
        a = int(rng.integers(0, tlen - qlen))
        q = synth.mutate(t[a : a + qlen], div, rng)
        out.append((f"hw{qlen}_{div}", np.ascontiguousarray(q, dtype=np.uint8), t))
    return out


def quirk_pairs():
    """a 3 Mbp pair at 0.5 %"""
    rng = np.random.default_rng(2028)
    t = synth.random_sequence(3_000_000, rng)
    q = synth.mutate(t, 0.005, rng)
    return [("3mbp", np.ascontiguousarray(q, dtype=np.uint8), t)]


def one_column_pair():
    """a 3.4 Mbp query against its first two bases: the Hirschberg split leaves a node of more than 3.36 Mbp against one
    target column, where edlib reads a column that does not exist (its result is undefined; in a test harness it can
    crash), so the device reports the distance and no path"""
    big = synth.random_sequence(3_400_000, np.random.default_rng(2030))
    return big, big[:2].copy()


# ---- the assembly-like CLI case ----------------------------------------------------------------------------------------

ASM_OPTS = ["-s", "10000", "--pi", "95"]
ASM_MODES = {"default": [], "one_to_one": ["-f", "one-to-one"]}


def write_asm(d):
    """three contigs of 1.2, 2.5 and 4 Mbp; the query a 0.5-2 % diverged copy with an inversion in the largest and a
    20 kb deletion in the middle one. Returns (reference FASTA, query FASTA)."""
    rng = np.random.default_rng(2029)
    genome = [synth.random_sequence(n, rng) for n in (1_200_000, 2_500_000, 4_000_000)]
    other = [synth.mutate(c, div, rng, ratio=(30, 2, 1)) for c, div in zip(genome, (0.005, 0.01, 0.02))]
    c = other[2]
    other[2] = np.concatenate([c[:1_500_000], synth.revcomp(c[1_500_000:1_800_000]), c[1_800_000:]])
    c = other[1]
    other[1] = np.concatenate([c[:1_000_000], c[1_020_000:]])
    ref, qry = os.path.join(d, "asm_ref.fa"), os.path.join(d, "asm_qry.fa")
    synth.write_fasta(ref, [f"r{i}" for i in range(3)], genome)
    synth.write_fasta(qry, [f"q{i}" for i in range(3)], other)
    return ref, qry


def paf_regions(paf_text, queries, refs):
    """(query region, target region) of every PAF line, cut and oriented as --align does"""
    for line in paf_text.splitlines():
        f = line.split("\t")
        qs, qe, ts, te = int(f[2]), int(f[3]), int(f[7]), int(f[8])
        q = queries[f[0]][qs:qe]
        if f[4] == "-":
            q = AD.revcomp(q)
        yield np.ascontiguousarray(q), np.ascontiguousarray(refs[f[5]][ts:te])
