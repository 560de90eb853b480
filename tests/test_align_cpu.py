"""mashmap-b200-align without a device: the full-matrix restatement of edlib's HW / PATH decisions against the unmodified
edlib (this pins the claim that a band-free computation takes edlib's decisions, DESIGN.md section 10), the C ABI's
declarations, the option parser and the job builder's loop semantics (--dryRun), and the stops where the reference
aligner fails an assert."""
import os
import re
import subprocess

import numpy as np
import pytest

import align_data as AD
from mashmap_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALIGN_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200-align")

needs_edlib = pytest.mark.skipif(not (AD.edlib_ref_available() and AD.oracle_available()),
                                 reason="oracle/_ref/libedlib_ref.so not built")


@needs_edlib
@pytest.mark.parametrize("seed", range(4))
def test_restatement_equals_edlib_on_random_pairs(seed):
    """4 x 2,600 pairs: lengths 1-2,000, 0-40 % error, repeats, homopolymers, N runs, a NUL at the target's end, k = -1,
    k = Q and k just around the distance; every 50th pair straddles the 1 MiB traceback / Hirschberg threshold"""
    rng = np.random.default_rng(1000 + seed)
    for i in range(2600):
        q, t = AD.random_pair(rng) if i % 50 else AD.threshold_pair(rng)
        k = AD.case_k(rng, q, t)
        a = AD.oracle_align(q, t, k)
        b = AD.edlib_ref_align(q, t, k)
        assert a[:3] == b[:3], (i, len(q), len(t), k)
        assert np.array_equal(a[3], b[3]), (i, len(q), len(t), k)
        if len(b[3]):
            assert AD.cigar(a[3]) == b[4]


@needs_edlib
def test_restatement_edge_cases():
    """k = 0, one-base inputs, no base in common with Q a multiple of 64 (edit distance Q, end 0), NUL against NUL.
    (With no base in common and Q not a multiple of 64, edlib's end is column -1 and edlib itself reads outside its
    buffers; the restatement and the device return the all-insertion path there.)"""
    cases = [(b"A", b"A", 0), (b"A", b"C", 0), (b"T" * 64, b"A" * 10, -1), (b"AC\x00", b"TTAC\x00", 1)]
    for q, t, k in cases:
        q, t = np.frombuffer(q, dtype=np.uint8).copy(), np.frombuffer(t, dtype=np.uint8).copy()
        a, b = AD.oracle_align(q, t, k), AD.edlib_ref_align(q, t, k)
        assert a[:3] == b[:3] and np.array_equal(a[3], b[3]), (q, t, k)


def test_align_abi_header_matches_exports():
    L = capi._align_lib()
    hdr = open(os.path.join(ROOT, "include", "mashmap_b200_align.h")).read()
    declared = set(re.findall(r"\b(mm_align_[a-z_0-9]+)\s*\(", hdr))
    assert declared == set(capi.ALIGN_EXPORTED_SYMBOLS)
    for s in declared:
        assert hasattr(L, s), s


def _w(path, text):
    with open(path, "w") as f:
        f.write(text)
    return path


@pytest.fixture
def tiny(tmp_path):
    d = str(tmp_path)
    _w(os.path.join(d, "ref.fa"), ">r1 desc\nACGTACGTAA\n>r2\nGGGGCCCCAA\n")
    _w(os.path.join(d, "q.fa"), ">a\nACGTAC\n>b\nGGGCC\n>c\nTTTT\n")
    return d


def _dry(d, mapping, *extra):
    p = subprocess.run([ALIGN_BIN, "-s", os.path.join(d, "ref.fa"), "-q", os.path.join(d, "q.fa"), "--mappingFile",
                        _w(os.path.join(d, "m.txt"), mapping), "--pi", "80", "--dryRun", *extra],
                       capture_output=True, text=True)
    jobs = [ln.split()[1:] for ln in p.stdout.splitlines() if ln.startswith("edlib ")]
    return p.returncode, jobs, p.stderr


def test_job_builder_walks_queries_and_lines_in_order(tiny):
    m = ("a 6 0 5 + r1 10 0 5 x\n"
         "a 6 1 4 - r1 10 2 6 x\n"
         "c 4 0 3 + r2 10 6 9 x\n"      # query b has no line: skipped; c matches
         "b 5 0 4 + r2 10 0 4 x\n")     # out of query order: lost, as in the reference
    rc, jobs, err = _dry(tiny, m)
    assert rc == 0, err
    assert [j[0] for j in jobs] == ["1", "2", "3"]
    assert jobs[1] == ["2", "a", "1", "4", "-", "r1", "2", "5", "0"]  # k = (int)((1 - 0.8f) * 4) = 0
    assert jobs[0][-1] == "1"                                          # (int)((1 - 0.8f) * 6) = 1 in float


def test_job_builder_line_that_matches_no_later_query_blocks_the_rest(tiny):
    rc, jobs, _ = _dry(tiny, "zz 6 0 5 + r1 10 0 5 x\na 6 0 5 + r1 10 0 5 x\n")
    assert rc == 0 and jobs == []


def test_job_builder_pi0_is_unbounded_and_nul_end_accepted(tiny):
    p = subprocess.run([ALIGN_BIN, "-s", os.path.join(tiny, "ref.fa"), "-q", os.path.join(tiny, "q.fa"), "--mappingFile",
                        _w(os.path.join(tiny, "m.txt"), "a 6 1 6 + r1 10 5 10 x\n"), "--pi", "0", "--dryRun"],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    job = [ln.split()[1:] for ln in p.stdout.splitlines() if ln.startswith("edlib ")][0]
    assert job == ["1", "a", "1", "6", "+", "r1", "5", "6", "-1"]


@pytest.mark.parametrize("line,what", [
    ("a 6 0 5 + r1 10 0\n", "fewer than 9 fields"),
    ("a 6 0 5 + r1 10 0 10\n", "subject region"),     # refLen 11 > 10: the reference's assert
    ("a 6 0 6 + r1 10 0 5\n", "query region"),        # queryLen 7 > 6
    ("a 6 3 7 + r1 10 0 4\n", "query region"),        # reads past the NUL
    ("a 6 0 5 + nope 10 0 5\n", "not in the subject"),
    ("a 6 x 5 + r1 10 0 5\n", "non-numeric"),
])
def test_job_builder_stops_where_the_reference_asserts(tiny, line, what):
    rc, jobs, err = _dry(tiny, line)
    assert rc == 1 and what in err and "mapping line 1" in err


def test_options(tiny):
    base = [ALIGN_BIN, "-s", os.path.join(tiny, "ref.fa"), "-q", os.path.join(tiny, "q.fa")]
    m = _w(os.path.join(tiny, "m.txt"), "a 6 0 5 + r1 10 0 5 x\n")
    assert subprocess.run(base + ["--pi", "80"], capture_output=True).returncode == 1              # no --mappingFile
    assert subprocess.run(base + ["--mappingFile", m], capture_output=True).returncode == 1        # no --pi
    assert subprocess.run(base + ["--mappingFile", m, "--pi", "80", "--bogus"], capture_output=True).returncode == 1
    ql = _w(os.path.join(tiny, "ql.txt"), os.path.join(tiny, "q.fa") + "\n" + os.path.join(tiny, "q.fa") + "\n")
    p = subprocess.run([ALIGN_BIN, "--sl", _w(os.path.join(tiny, "sl.txt"), os.path.join(tiny, "ref.fa") + "\n"),
                        "--ql", ql, "--mappingFile", m, "--perc_identity=80", "-t", "4", "-o", "x.sam", "--dryRun"],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert sum(ln.startswith("edlib ") for ln in p.stdout.splitlines()) == 2  # the mapping file re-opened per query file
    assert subprocess.run([ALIGN_BIN, "-h"], capture_output=True).returncode == 0
