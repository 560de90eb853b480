"""Test-side helpers for mashmap-b200-align: the random pair generator, ctypes views of the two CPU checkers
(oracle/libalign_oracle.so, the full-matrix restatement, and oracle/_ref/libedlib_ref.so, the unmodified edlib), and the
CIGAR text of an edit-op list. Test infrastructure only."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "libalign_oracle.so")
EDLIB_REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libedlib_ref.so")
ALIGN_REF_BIN = os.path.join(ROOT, "oracle", "_ref", "mashmap_align_ref")
MAP_REF_BIN = os.path.join(ROOT, "oracle", "_ref", "mashmap_ref")

_ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
_COMP = np.arange(256, dtype=np.uint8)
for _a, _b in zip(b"ACGT", b"TGCA"):
    _COMP[_a] = _b


def revcomp(a):
    """CommonFunc::reverseComplement: ACGT complemented, every other byte (N, NUL) kept"""
    return _COMP[np.asarray(a, dtype=np.uint8)[::-1]]


def _mutate(seq, err, rng):
    out = []
    for b in seq:
        r = rng.random()
        if r < err * 0.4:
            out.append(int(_ACGT[rng.integers(4)]))
        elif r < err * 0.7:
            out.append(int(b))
            out.append(int(_ACGT[rng.integers(4)]))
        elif r < err:
            pass
        else:
            out.append(int(b))
    return np.array(out, dtype=np.uint8)


def random_pair(rng, max_len=2000):
    """One (query, target, k) case. Kinds: random pairs at 0-40 % error, tandem repeats and homopolymers (many tie
    paths), N runs, a NUL at the target's end, and k just below / at / above the true distance or k = -1 (the last two
    are chosen by the caller, who knows the distance)."""
    kind = int(rng.integers(6))
    n = int(rng.integers(1, max_len + 1)) if rng.random() < 0.7 else int(rng.integers(1, 64))
    if kind == 0:  # random region of a random target
        src = _ACGT[rng.integers(0, 4, size=n)]
    elif kind == 1:  # tandem repeat
        unit = _ACGT[rng.integers(0, 4, size=int(rng.integers(1, 8)))]
        src = np.resize(unit, n)
    elif kind == 2:  # homopolymer runs
        src = np.repeat(_ACGT[rng.integers(0, 4, size=n)], rng.integers(1, 12, size=n))[:n]
    elif kind == 3:  # N runs
        src = _ACGT[rng.integers(0, 4, size=n)].copy()
        for _ in range(int(rng.integers(1, 4))):
            a = int(rng.integers(0, n)); src[a : a + int(rng.integers(1, 40))] = ord("N")
    else:
        src = _ACGT[rng.integers(0, 4, size=n)]
    err = float(rng.uniform(0, 0.4))
    q = _mutate(src, err, rng)
    if len(q) == 0:
        q = src[:1].copy()
    flank = int(rng.integers(0, 200))
    left = _ACGT[rng.integers(0, 4, size=int(rng.integers(0, flank + 1)))]
    right = _ACGT[rng.integers(0, 4, size=flank - len(left))]
    t = np.concatenate([left, src, right]).astype(np.uint8)
    if kind == 5 or rng.random() < 0.05:  # the terminating NUL a v3 end coordinate pulls in
        t = np.concatenate([t, np.zeros(1, dtype=np.uint8)])
        if rng.random() < 0.5:
            q = np.concatenate([q, np.zeros(1, dtype=np.uint8)])
    if rng.random() < 0.1:
        q = revcomp(q)
    return np.ascontiguousarray(q, dtype=np.uint8), np.ascontiguousarray(t, dtype=np.uint8)


def threshold_pair(rng):
    """A pair whose NW path problem sits near edlib's 1 MiB traceback / Hirschberg threshold:
    20 * ceil(Q / 64) * T + 8 * T ~ 2^20."""
    Q = int(rng.integers(1500, 2001))
    nb = (Q + 63) // 64
    T0 = (1 << 20) // (20 * nb + 8)
    src = _ACGT[rng.integers(0, 4, size=T0 + int(rng.integers(-3, 4)))]
    q = _mutate(src, float(rng.uniform(0, 0.15)), rng)
    return np.ascontiguousarray(q[: max(1, len(q))]), np.ascontiguousarray(src)


_ora = None
_ref = None


def oracle_available():
    return os.path.exists(ORACLE_LIB)


def edlib_ref_available():
    return os.path.exists(EDLIB_REF_LIB)


def oracle_align(q, t, k):
    """(ed, start, end, ops) of the full-matrix restatement"""
    global _ora
    if _ora is None:
        _ora = C.CDLL(ORACLE_LIB)
        _ora.ora_align.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 5
    ed, st, en, n = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    ops = np.zeros(len(q) + len(t) + 1, dtype=np.uint8)
    _ora.ora_align(q.ctypes.data, len(q), t.ctypes.data, len(t), int(k), C.byref(ed), C.byref(st), C.byref(en),
                   ops.ctypes.data, C.byref(n))
    return ed.value, st.value, en.value, ops[: n.value].copy()


def edlib_ref_align(q, t, k):
    """(ed, start, end, ops, cigar) of the unmodified edlib"""
    global _ref
    if _ref is None:
        _ref = C.CDLL(EDLIB_REF_LIB)
        _ref.ref_edlib_align.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int]
    ed, st, en, n = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    ops = np.zeros(len(q) + len(t) + 1, dtype=np.uint8)
    cig = C.create_string_buffer(4 * (len(q) + len(t)) + 16)
    _ref.ref_edlib_align(q.ctypes.data, len(q), t.ctypes.data, len(t), int(k), C.byref(ed), C.byref(st), C.byref(en),
                         ops.ctypes.data, C.byref(n), cig, len(cig))
    return ed.value, st.value, en.value, ops[: n.value].copy(), cig.value.decode()


def cigar(ops):
    """EDLIB_CIGAR_STANDARD text of an edit-op list (0 match, 1 I, 2 D, 3 mismatch -> M I D M)"""
    ch = "MIDM"
    out, last, run = [], None, 0
    for o in np.asarray(ops).tolist():
        c = ch[o]
        if c == last:
            run += 1
        else:
            if last is not None:
                out.append(f"{run}{last}")
            last, run = c, 1
    if last is not None:
        out.append(f"{run}{last}")
    return "".join(out)


def case_k(rng, q, t):
    """k for a case: -1, a large bound, or just around the true distance (needs the oracle)"""
    r = rng.random()
    if r < 0.2:
        return -1
    if r < 0.4:
        return len(q)
    ed = oracle_align(q, t, -1)[0]
    return max(0, ed + int(rng.integers(-2, 3)))
