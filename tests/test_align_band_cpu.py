"""The static band of long NW sub-problems without a device: a full-matrix restatement restricted to the band
(ora_align_band_nw, oracle/align_band_oracle.cpp, cells outside the band at +infinity) takes the same decisions as the
band-free restatement (ora_align_nw): the distance with edlib's k rule and every Hirschberg split row of banded columns
at the node's exact score (DESIGN.md section 10). Also the routing constant of include/mashmap_b200_align.h."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import align_data as AD
import align_nw_data as AN
from mashmap_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAND_LIB = os.path.join(ROOT, "oracle", "libalign_band_oracle.so")

_lib = None


def band_align_nw(q, t, k):
    """(ed, start, end, ops) of the static-band restatement"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(BAND_LIB)
        _lib.ora_align_band_nw.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 5
    ed, st, en, n = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    ops = np.zeros(len(q) + len(t) + 1, dtype=np.uint8)
    _lib.ora_align_band_nw(q.ctypes.data, len(q), t.ctypes.data, len(t), int(k), C.byref(ed), C.byref(st),
                           C.byref(en), ops.ctypes.data, C.byref(n))
    return ed.value, st.value, en.value, ops[: n.value].copy()


def _len_mod64_pair(rng):
    """a close pair whose query length is 0, 1 or 63 mod 64 (a full, a nearly empty and a nearly full last block)"""
    n = 64 * int(rng.integers(1, 31)) + int(rng.choice([0, 1, -1]))
    src = AD._ACGT[rng.integers(0, 4, size=n + 40)]
    q = AD._mutate(src, float(rng.uniform(0, 0.1)), rng)
    q = np.resize(q, n) if len(q) >= n else np.concatenate([q, src[: n - len(q)]])
    return np.ascontiguousarray(q, dtype=np.uint8), np.ascontiguousarray(src)


def _k(rng, q, t, ed):
    r = rng.random()
    if r < 0.25:
        return -1
    if r < 0.45:
        return ed
    if r < 0.6:
        return max(0, ed - 1)
    if r < 0.7:  # below the length difference: decided without a pass
        return max(0, abs(len(q) - len(t)) - 1 - int(rng.integers(0, 3)))
    return ed + int(rng.integers(1, 40))


@pytest.mark.parametrize("seed", range(4))
def test_band_restatement_equals_full_matrix(seed):
    """4 x 2,600 pairs: the CPU tests' generators (lengths 1-2,000, repeats, homopolymers, N runs, a NUL at the end),
    long indels, query lengths 0 / 1 / 63 mod 64 and pairs above the 1 MiB traceback / Hirschberg threshold (whose
    split rows come from banded columns); k = -1, k = ed, ed - 1, above ed and below |Q - T|"""
    rng = np.random.default_rng(9100 + seed)
    n_hirsch = n_none = n_exact_k = 0
    for i in range(2600):
        if i % 40 == 0:
            q, t = AD.threshold_pair(rng)
        elif i % 7 == 0:
            q, t = AN.long_indel_pair(rng)
        elif i % 5 == 0:
            q, t = _len_mod64_pair(rng)
        else:
            q, t = AD.random_pair(rng)
        ed = AN.oracle_align_nw(q, t, -1)[0]
        k = _k(rng, q, t, ed)
        a = band_align_nw(q, t, k)
        b = AN.oracle_align_nw(q, t, k)
        assert a[:3] == b[:3], (seed, i, len(q), len(t), k)
        assert np.array_equal(a[3], b[3]), (seed, i, len(q), len(t), k)
        n_none += b[0] < 0
        n_exact_k += k == ed
        nb = (len(q) + 63) // 64
        n_hirsch += b[0] >= 0 and 20 * nb * len(t) + 8 * len(t) >= 1 << 20
    assert n_none > 300 and n_exact_k > 300 and n_hirsch > 30


def test_band_restatement_edge_cases():
    """one-base inputs, k = 0, a length difference at / just above k, a zero-width band (k = |Q - T|), tandem repeats
    with many co-optimal paths above the Hirschberg threshold, N runs"""
    rng = np.random.default_rng(17)
    unit = np.frombuffer(b"ACG", dtype=np.uint8)
    rep = np.resize(unit, 1900)
    cases = [(b"A", b"A", 0), (b"A", b"C", 0), (b"A", b"C", -1), (b"T" * 64, b"A" * 10, 54), (b"T" * 64, b"A" * 10, 63),
             (b"ACGT", b"ACGTACG", 3), (b"ACGT", b"ACGTACG", 2), (b"N" * 70, b"N" * 5, -1)]
    cases = [(np.frombuffer(q, dtype=np.uint8).copy(), np.frombuffer(t, dtype=np.uint8).copy(), k) for q, t, k in cases]
    cases += [(rep[:1800].copy(), rep.copy(), -1), (rep[:1800].copy(), rep.copy(), 100), (rep.copy(), rep[5:].copy(), 5)]
    src = AD._ACGT[rng.integers(0, 4, size=1950)]
    cases += [(np.concatenate([src[:900], src[1000:]]), src.copy(), k) for k in (-1, 100, 99)]
    for q, t, k in cases:
        a, b = band_align_nw(q, t, k), AN.oracle_align_nw(q, t, k)
        assert a[:3] == b[:3] and np.array_equal(a[3], b[3]), (len(q), len(t), k)


def test_band_min_len_is_in_the_header_and_capi():
    hdr = open(os.path.join(ROOT, "include", "mashmap_b200_align.h")).read()
    m = re.search(r"#define MM_ALIGN_BAND_MIN_LEN \((\d+) \* (\d+)\)", hdr)
    assert m, "MM_ALIGN_BAND_MIN_LEN missing from the header"
    assert int(m.group(1)) * int(m.group(2)) == capi.MM_ALIGN_BAND_MIN_LEN == 32768
    assert capi.MM_ALIGN_BAND_MIN_LEN > 12_000  # the 10 kb reads of scripts/map_align_perf.py stay on the warp path
