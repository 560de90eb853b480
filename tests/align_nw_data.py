"""Test-side helpers for edlib's global mode (EDLIB_MODE_NW), the alignment mashmap-b200 --align writes: ctypes views of the
NW entry points of the two CPU checkers (ora_align_nw in oracle/libalign_nw_oracle.so, the full-matrix restatement, and
ref_edlib_align_nw in oracle/_ref/libedlib_nw_ref.so, the unmodified edlib; both built by oracle/align_nw.mk), and the
check of a PAF file's NM:i / cg:Z tags against regions cut from the FASTA files in Python. Test infrastructure only."""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np

import align_data as AD

ORACLE_NW_LIB = os.path.join(AD.ROOT, "oracle", "libalign_nw_oracle.so")
EDLIB_NW_REF_LIB = os.path.join(AD.ROOT, "oracle", "_ref", "libedlib_nw_ref.so")

_ora = None
_ref = None


def oracle_nw_available():
    return os.path.exists(ORACLE_NW_LIB)


def edlib_nw_ref_available():
    return os.path.exists(EDLIB_NW_REF_LIB)


def oracle_align_nw(q, t, k):
    """(ed, start, end, ops) of the full-matrix restatement of edlibAlign(NW, PATH)"""
    global _ora
    if _ora is None:
        _ora = C.CDLL(ORACLE_NW_LIB)
        _ora.ora_align_nw.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 5
    ed, st, en, n = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    ops = np.zeros(len(q) + len(t) + 1, dtype=np.uint8)
    _ora.ora_align_nw(q.ctypes.data, len(q), t.ctypes.data, len(t), int(k), C.byref(ed), C.byref(st), C.byref(en),
                      ops.ctypes.data, C.byref(n))
    return ed.value, st.value, en.value, ops[: n.value].copy()


def edlib_ref_align_nw(q, t, k):
    """(ed, start, end, ops, cigar) of the unmodified edlibAlign(NW, PATH)"""
    global _ref
    if _ref is None:
        _ref = C.CDLL(EDLIB_NW_REF_LIB)
        _ref.ref_edlib_align_nw.argtypes = ([C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 6
                                            + [C.c_int])
    ed, st, en, n = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    ops = np.zeros(len(q) + len(t) + 1, dtype=np.uint8)
    cig = C.create_string_buffer(4 * (len(q) + len(t)) + 16)
    _ref.ref_edlib_align_nw(q.ctypes.data, len(q), t.ctypes.data, len(t), int(k), C.byref(ed), C.byref(st),
                            C.byref(en), ops.ctypes.data, C.byref(n), cig, len(cig))
    return ed.value, st.value, en.value, ops[: n.value].copy(), cig.value.decode()


def nw_check():
    """the NW checker to compare with: the unmodified edlib where it is built, the restatement otherwise"""
    return edlib_ref_align_nw if edlib_nw_ref_available() else oracle_align_nw


def long_indel_pair(rng):
    """a pair whose lengths differ by more than the k the caller picks around the distance: a long insertion or
    deletion in an otherwise close copy"""
    n = int(rng.integers(50, 1500))
    src = AD._ACGT[rng.integers(0, 4, size=n)]
    gap = AD._ACGT[rng.integers(0, 4, size=int(rng.integers(65, 400)))]
    at = int(rng.integers(0, n + 1))
    long = np.concatenate([src[:at], gap, src[at:]]).astype(np.uint8)
    q = AD._mutate(src, float(rng.uniform(0, 0.1)), rng)
    if len(q) == 0:
        q = src[:1].copy()
    return (np.ascontiguousarray(q), long) if rng.random() < 0.5 else (long, np.ascontiguousarray(q))


def case_k_nw(rng, q, t):
    """k for an NW case: -1, a large bound, or just around the true NW distance"""
    r = rng.random()
    if r < 0.25:
        return -1
    if r < 0.4:
        return max(len(q), len(t))
    ed = oracle_align_nw(q, t, -1)[0]
    return max(0, ed + int(rng.integers(-2, 3)))


# ---- a PAF file's tags against the FASTA files ----------------------------------------------------------------------

_NORM = np.full(256, ord("N"), dtype=np.uint8)
for _c in b"ACGT":
    _NORM[_c] = _c
    _NORM[_c + 32] = _c


def read_fasta(path):
    """name (header up to the first space) -> normalised bases (upper case ACGT, everything else N) as uint8"""
    out, name, parts = {}, None, []
    with open(path, "rb") as f:
        for line in f:
            line = line.rstrip(b"\n")
            if line.startswith(b">"):
                if name is not None:
                    out[name] = _NORM[np.frombuffer(b"".join(parts), dtype=np.uint8)]
                name, parts = line[1:].split(b" ")[0].decode(), []
            else:
                parts.append(line)
    if name is not None:
        out[name] = _NORM[np.frombuffer(b"".join(parts), dtype=np.uint8)]
    return out


def strip_tags(text):
    """the PAF text without the NM:i / cg:Z tags --align appends"""
    return re.sub(r"\tNM:i:[0-9]+\tcg:Z:[0-9MID]*(?=\n)", "", text)


def cigar_lengths(cg):
    """(query bases, target bases) a standard CIGAR consumes"""
    q = t = 0
    for n, op in re.findall(r"([0-9]+)([MID])", cg):
        n = int(n)
        q += n if op in "MI" else 0
        t += n if op in "MD" else 0
    return q, t


def check_tags(paf_text, queries, refs, max_len=None, check=None):
    """Every line of an --align PAF: its CIGAR consumes exactly its query and target region, and NM / cg equal edlib NW
    (or the restatement) of the regions cut here; lines over max_len carry no tags. Returns (tagged, untagged)."""
    check = check or nw_check()
    tagged = untagged = 0
    for line in paf_text.splitlines():
        f = line.split("\t")
        qs, qe, ts, te = int(f[2]), int(f[3]), int(f[7]), int(f[8])
        tags = {x[:4]: x[5:] for x in f[12:] if x[:4] in ("NM:i", "cg:Z")}
        if max_len is not None and max(qe - qs, te - ts) > max_len:
            assert not tags, line
            untagged += 1
            continue
        assert set(tags) == {"NM:i", "cg:Z"} and f[-2].startswith("NM:i:") and f[-1].startswith("cg:Z:"), line
        assert cigar_lengths(tags["cg:Z"]) == (qe - qs, te - ts), line
        q = queries[f[0]][qs:qe]
        if f[4] == "-":
            q = AD.revcomp(q)
        t = refs[f[5]][ts:te]
        want = check(np.ascontiguousarray(q), np.ascontiguousarray(t), -1)
        assert int(tags["NM:i"]) == want[0], line[:200]
        assert tags["cg:Z"] == AD.cigar(want[3]), line[:200]
        tagged += 1
    return tagged, untagged
