"""Test-side restatement of the tag text mashmap-b200 --align --eqx / --cs writes, from an edit-op path (0 match,
1 insertion, 2 deletion, 3 mismatch) and the query / target it aligns: edlibAlignmentToCigar's standard and extended
CIGARs, minimap2's short cs string, the inverse operations the tests use to check them (collapse an extended CIGAR, apply
a cs string to the target), and the check of a PAF file's three tags against regions cut from the FASTA files. Test
infrastructure only."""
from __future__ import annotations

import re

import numpy as np

import align_data as AD
import align_nw_data as AN

_LOWER = np.arange(256, dtype=np.uint8)
_LOWER[ord("A") : ord("Z") + 1] += 32


def lower(a):
    """bytes with A-Z lowered to a-z, every other byte kept"""
    a = np.frombuffer(a, dtype=np.uint8) if isinstance(a, (bytes, bytearray)) else np.asarray(a, dtype=np.uint8)
    return _LOWER[a].tobytes()


def runs(ops, fold_mismatch):
    """[(op, length)] of maximal runs of one letter; with fold_mismatch a mismatch counts as a match (letter M)"""
    o = np.asarray(ops, dtype=np.uint8)
    if len(o) == 0:
        return []
    key = np.where(o == 3, 0, o) if fold_mismatch else o
    starts = np.flatnonzero(np.concatenate([[True], key[1:] != key[:-1]]))
    ends = np.concatenate([starts[1:], [len(o)]])
    return [(int(key[s]), int(e - s)) for s, e in zip(starts, ends)]


def cigar_std(ops):
    """edlibAlignmentToCigar(EDLIB_CIGAR_STANDARD)"""
    return "".join(f"{n}{'MIDM'[op]}" for op, n in runs(ops, True))


def cigar_eqx(ops):
    """edlibAlignmentToCigar(EDLIB_CIGAR_EXTENDED)"""
    return "".join(f"{n}{'=IDX'[op]}" for op, n in runs(ops, False))


def cs_short(ops, q, t):
    """minimap2's short cs of the path: ':N' per match run, '*tq' per mismatch, '+bases' / '-bases' per insertion /
    deletion run; bases lowered"""
    q, t = lower(q), lower(t)
    out, i, j = [], 0, 0
    for op, n in runs(ops, False):
        if op == 0:
            out.append(f":{n}")
            i, j = i + n, j + n
        elif op == 3:
            out.append(b"".join(b"*" + t[j + m : j + m + 1] + q[i + m : i + m + 1] for m in range(n)).decode("latin1"))
            i, j = i + n, j + n
        elif op == 1:
            out.append("+" + q[i : i + n].decode("latin1"))
            i += n
        else:
            out.append("-" + t[j : j + n].decode("latin1"))
            j += n
    assert (i, j) == (len(q), len(t))
    return "".join(out)


def collapse(eqx):
    """an extended CIGAR with = / X folded into M"""
    out, last, run = [], None, 0
    for n, op in re.findall(r"([0-9]+)([=XIDM])", eqx):
        op = "M" if op in "=X" else op
        if op == last:
            run += int(n)
        else:
            if last is not None:
                out.append(f"{run}{last}")
            last, run = op, int(n)
    if last is not None:
        out.append(f"{run}{last}")
    return "".join(out)


def eqx_differences(eqx):
    """X + I + D bases of an extended CIGAR: the edit distance of its path"""
    return sum(int(n) for n, op in re.findall(r"([0-9]+)([XID])", eqx))


_CS = re.compile(r":([0-9]+)|\*(.)(.)|\+([^:*+\-]+)|-([^:*+\-]+)", re.S)


def cs_differences(cs):
    """mismatches + inserted + deleted bases of a cs string"""
    n = 0
    for m in _CS.finditer(cs):
        n += 1 if m.group(2) is not None else len(m.group(4) or m.group(5) or "")
    return n


def apply_cs(cs, t):
    """the query a cs string makes of the target t (lowered); asserts that the string's target bases are t's and that
    it consumes t exactly"""
    t = lower(t)
    out, j, pos = [], 0, 0
    for m in _CS.finditer(cs):
        assert m.start() == pos, (cs[pos : pos + 20], pos)
        pos = m.end()
        if m.group(1) is not None:
            n = int(m.group(1))
            assert n > 0
            out.append(t[j : j + n])
            j += n
        elif m.group(2) is not None:
            assert m.group(2) != m.group(3) and t[j : j + 1] == m.group(2).encode("latin1"), (j, m.group(0))
            out.append(m.group(3).encode("latin1"))
            j += 1
        elif m.group(4) is not None:
            out.append(m.group(4).encode("latin1"))
        else:
            d = m.group(5).encode("latin1")
            assert t[j : j + len(d)] == d, (j, m.group(0))
            j += len(d)
    assert pos == len(cs) and j == len(t), (pos, len(cs), j, len(t))
    return b"".join(out)


def check_tag_paf(text, plain, queries, refs, max_len=None):
    """An --align --eqx --cs PAF against the plain --align PAF of the same run: columns 1-12 and NM:i equal, cg:Z
    collapses to plain's cg:Z, its X + I + D is NM, and cs:Z applied to the target region cut from the FASTA gives the
    query region (reverse-complemented on '-'). Lines over max_len carry none of the three tags. Returns (tagged,
    untagged)."""
    a, b = text.splitlines(), plain.splitlines()
    assert len(a) == len(b)
    tagged = untagged = 0
    for la, lb in zip(a, b):
        fa, fb = la.split("\t"), lb.split("\t")
        assert fa[:12] == fb[:12], la[:200]
        qs, qe, ts, te = int(fa[2]), int(fa[3]), int(fa[7]), int(fa[8])
        if max_len is not None and max(qe - qs, te - ts) > max_len:
            assert not any(x[:5] in ("NM:i:", "cg:Z:", "cs:Z:") for x in fa[12:]), la[:200]
            assert la == lb
            untagged += 1
            continue
        assert fa[-3].startswith("NM:i:") and fa[-2].startswith("cg:Z:") and fa[-1].startswith("cs:Z:"), la[:200]
        assert fa[12:-3] == fb[12:-2] and fa[-3] == fb[-2], la[:200]
        eqx, cs = fa[-2][5:], fa[-1][5:]
        assert collapse(eqx) == fb[-1][5:], la[:200]
        assert eqx_differences(eqx) == int(fa[-3][5:]), la[:200]
        q = queries[fa[0]][qs:qe]
        if fa[4] == "-":
            q = AD.revcomp(q)
        assert apply_cs(cs, refs[fa[5]][ts:te]) == lower(q), la[:200]
        tagged += 1
    return tagged, untagged


def tag_pairs(rng, n):
    """identity 60-100 %, long indels, N runs, one-base sides, and the CPU tests' general generator"""
    out = []
    for i in range(n):
        kind = i % 5
        if kind == 0:
            src = AD._ACGT[rng.integers(0, 4, size=int(rng.integers(1, 1500)))]
            q = AD._mutate(src, float(rng.uniform(0, 0.4)), rng)
            q = q if len(q) else src[:1].copy()
            out.append((np.ascontiguousarray(q, dtype=np.uint8), src.astype(np.uint8)))
        elif kind == 1:
            out.append(AN.long_indel_pair(rng))
        elif kind == 2:  # N runs on both sides, N against N is a match
            src = AD._ACGT[rng.integers(0, 4, size=int(rng.integers(50, 800)))].copy()
            a = int(rng.integers(0, len(src) - 10))
            src[a : a + int(rng.integers(1, 10))] = ord("N")
            q = AD._mutate(src, float(rng.uniform(0, 0.2)), rng)
            q = q if len(q) else src[:1].copy()
            out.append((np.ascontiguousarray(q, dtype=np.uint8), src.astype(np.uint8)))
        elif kind == 3:  # a one-base side
            one = AD._ACGT[rng.integers(0, 4, size=1)].astype(np.uint8)
            other = AD._ACGT[rng.integers(0, 4, size=int(rng.integers(1, 200)))].astype(np.uint8)
            out.append((one, other) if rng.random() < 0.5 else (other, one))
        else:
            out.append(AD.random_pair(rng)[:2])
    return out


def edlib_or_oracle(q, t):
    """(ed, ops, standard cigar) of edlib NW with k = -1 where it is built, of the restatement otherwise"""
    if AN.edlib_nw_ref_available():
        r = AN.edlib_ref_align_nw(q, t, -1)
        return r[0], r[3], r[4]
    r = AN.oracle_align_nw(q, t, -1)
    return r[0], r[3], AD.cigar(r[3])
