"""mashmap-b200 --align without a device: the full-matrix restatement of edlib's global mode (NW, PATH) against the
unmodified edlib (this pins the claim that a band-free computation takes edlib's NW decisions, DESIGN.md section 10),
the options --align refuses, and the mm_align_job layout."""
import os
import re
import subprocess

import numpy as np
import pytest

import align_data as AD
import align_nw_data as AN
from mashmap_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAP_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200")

needs_edlib = pytest.mark.skipif(not (AN.edlib_nw_ref_available() and AN.oracle_nw_available()),
                                 reason="oracle/_ref/libedlib_nw_ref.so not built")


@needs_edlib
@pytest.mark.parametrize("seed", range(4))
def test_nw_restatement_equals_edlib_on_random_pairs(seed):
    """4 x 2,600 pairs: lengths 1-2,000 at 0-40 % error, repeats, homopolymers, N runs, a NUL at the end; every 7th pair
    has a length difference above the k picked around its distance; k = -1, a large k and k just around the distance;
    every 50th pair straddles the 1 MiB traceback / Hirschberg threshold"""
    rng = np.random.default_rng(5000 + seed)
    n_below = 0
    for i in range(2600):
        if i % 50 == 0:
            q, t = AD.threshold_pair(rng)
        elif i % 7 == 0:
            q, t = AN.long_indel_pair(rng)
        else:
            q, t = AD.random_pair(rng)
        k = AN.case_k_nw(rng, q, t)
        a = AN.oracle_align_nw(q, t, k)
        b = AN.edlib_ref_align_nw(q, t, k)
        assert a[:3] == b[:3], (i, len(q), len(t), k)
        assert np.array_equal(a[3], b[3]), (i, len(q), len(t), k)
        if b[0] >= 0:
            assert b[1:3] == (0, len(t) - 1) and AD.cigar(a[3]) == b[4]
            assert AN.cigar_lengths(b[4]) == (len(q), len(t))
        else:
            n_below += 1
    assert n_below > 100  # k below the distance, length differences above k included


@needs_edlib
def test_nw_restatement_edge_cases():
    """one-base inputs, k = 0, no base in common, a length difference just above / at k, NUL against NUL"""
    cases = [(b"A", b"A", 0), (b"A", b"C", 0), (b"A", b"C", -1), (b"T" * 64, b"A" * 10, -1), (b"T" * 70, b"A", -1),
             (b"ACGT", b"ACGTACG", 2), (b"ACGT", b"ACGTACG", 3), (b"AC\x00", b"TTAC\x00", 1), (b"N" * 5, b"N" * 5, 0)]
    for q, t, k in cases:
        q, t = np.frombuffer(q, dtype=np.uint8).copy(), np.frombuffer(t, dtype=np.uint8).copy()
        a, b = AN.oracle_align_nw(q, t, k), AN.edlib_ref_align_nw(q, t, k)
        assert a[:3] == b[:3] and np.array_equal(a[3], b[3]), (q, t, k)


def _w(path, text):
    with open(path, "w") as f:
        f.write(text)
    return path


def test_align_legacy_is_refused_before_the_reference_is_read(tmp_path):
    q = _w(str(tmp_path / "q.fa"), ">q\nACGT\n")
    p = subprocess.run([MAP_BIN, "-r", str(tmp_path / "missing.fa"), "-q", q, "--align", "--legacy"],
                       capture_output=True, text=True)
    assert p.returncode == 1 and "--legacy" in p.stderr and "Could not open" not in p.stderr, p.stderr


@pytest.mark.parametrize("value", ["0", "-5", "abc", "1e6", "", "99999999999"])
def test_invalid_align_max_len_is_refused(tmp_path, value):
    r = _w(str(tmp_path / "r.fa"), ">r\nACGT\n")
    p = subprocess.run([MAP_BIN, "-r", r, "-q", r, "--align", "--alignMaxLen", value], capture_output=True, text=True)
    assert p.returncode == 1 and "--alignMaxLen" in p.stderr, p.stderr


def test_align_max_len_needs_align(tmp_path):
    r = _w(str(tmp_path / "r.fa"), ">r\nACGT\n")
    p = subprocess.run([MAP_BIN, "-r", r, "-q", r, "--alignMaxLen", "100"], capture_output=True, text=True)
    assert p.returncode == 1 and "--alignMaxLen" in p.stderr and "--align" in p.stderr, p.stderr


def test_align_job_layout_is_unchanged_apart_from_the_mode_field():
    d = capi.align_job_dtype
    assert d.itemsize == 32
    assert [(n, d.fields[n][0].str, d.fields[n][1]) for n in d.names] == [
        ("q_offset", "<u8", 0), ("t_offset", "<u8", 8), ("q_len", "<i4", 16), ("t_len", "<i4", 20), ("k", "<i4", 24),
        ("mode", "<i4", 28)]
    hdr = open(os.path.join(ROOT, "include", "mashmap_b200_align.h")).read()
    body = re.search(r"typedef struct mm_align_job \{(.*?)\} mm_align_job;", hdr, re.S).group(1)
    assert re.findall(r"(\w+)\s+(\w+);", body) == [("uint64_t", "q_offset"), ("uint64_t", "t_offset"),
                                                   ("int32_t", "q_len"), ("int32_t", "t_len"), ("int32_t", "k"),
                                                   ("int32_t", "mode")]
    modes = dict(re.findall(r"#define (MM_ALIGN_\w+) (\d+)", hdr))
    assert modes == {"MM_ALIGN_HW": str(capi.MM_ALIGN_HW), "MM_ALIGN_NW": str(capi.MM_ALIGN_NW)} == {
        "MM_ALIGN_HW": "0", "MM_ALIGN_NW": "1"}
