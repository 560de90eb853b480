"""The reference index built ON THE DEVICE (mm_index_build, SURVEY 8(f)-1) against the index the UNMODIFIED reference builds
(oracle/_ref harness: Sketch::build / index / computeFreqHist / dropFreqSeedSet): minmerIndex after the frequent-seed drop,
the lookup keys / interval points, the frequent-seed flags and the threshold. Records must be the reference's; the one
permitted difference is the order of records with equal (seqId, wpos, wpos_end), which the reference leaves to std::sort's
unspecified tie order (commonFunc.hpp:558) and the device builder keeps in emission order (DESIGN.md). Where the reference
is not built, the device index is compared with the reference's stored digests (golden_ref.py)."""
import os

import numpy as np
import pytest

import datasets
import golden_ref
import refh
from conftest import have_gpu
from mashmap_b200 import synth

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not have_gpu(), reason="no GPU")]


def canon_minmers(mi):
    """records grouped by (seqId, wpos, wpos_end): the groups in order, each group as a sorted list (tie order is free)"""
    key = np.stack([mi["seqId"].astype(np.int64), mi["wpos"].astype(np.int64), mi["wpos_end"].astype(np.int64)], axis=1)
    assert np.all(np.lexsort((key[:, 2], key[:, 1], key[:, 0])) == np.arange(len(key))) or _is_sorted(key), "not sorted by (seqId, wpos, wpos_end)"
    out, i = [], 0
    rows = list(zip(key[:, 0].tolist(), key[:, 1].tolist(), key[:, 2].tolist(), mi["hash"].tolist(), mi["strand"].tolist()))
    while i < len(rows):
        j = i
        while j < len(rows) and rows[j][:3] == rows[i][:3]:
            j += 1
        out.append(sorted(rows[i:j]))
        i = j
    return out


def _is_sorted(key):
    a = key[:-1]
    b = key[1:]
    return bool(np.all((a[:, 0] < b[:, 0]) | ((a[:, 0] == b[:, 0]) & ((a[:, 1] < b[:, 1]) | ((a[:, 1] == b[:, 1]) & (a[:, 2] <= b[:, 2]))))))


def lookup_dict(keys, offs, pts, fr):
    d = {}
    for i, k in enumerate(keys.tolist()):
        p = pts[int(offs[i]) : int(offs[i + 1])]
        d[k] = (list(zip(p["pos"].tolist(), p["seqId"].tolist(), p["side"].tolist())), int(fr[i]))
    return d


def build_and_compare(d, args, chunk=None, monkeypatch=None, expect_fixed=None):
    from mashmap_b200 import capi

    if chunk is not None:
        monkeypatch.setenv("MM_INDEX_CHUNK", str(chunk))
    if not refh.available():
        return build_and_compare_stored(d, args, expect_fixed)
    R = refh.RefSession(args)
    golden_ref.check_stored("sessions", golden_ref.key_of(args, d), golden_ref.session_digests(R))
    try:
        ctx = capi.Context(kmer_size=R.p.kmerSize, seg_length=R.p.segLength, sketch_size=R.p.sketchSize)
        seqs = np.concatenate(d["genome"]).astype(np.uint8)
        offs = np.zeros(len(d["genome"]) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(c) for c in d["genome"]])
        st = ctx.index_build(seqs, offs, kmer_pct_threshold=float(R.p.kmer_pct_threshold), keep_lookup=True)
        print("device index:", st)
        mi, keys, ko, pts, fr = ctx.index_download()
        ref_mi = R.index()
        rk, ro, rp, rf = R.lookup()
        assert st["freq_threshold"] == R.freq_threshold()
        assert len(mi) == len(ref_mi), (len(mi), len(ref_mi))
        a, b = canon_minmers(mi), canon_minmers(ref_mi)
        assert a == b
        ties = sum(len(g) > 1 for g in a)
        same_order = all(np.array_equal(mi[f], ref_mi[f]) for f in ("hash", "wpos", "wpos_end", "seqId", "strand"))
        print(f"{len(mi)} minmers, {ties} groups of exact (seqId, wpos, wpos_end) ties, identical order: {same_order}")
        assert np.array_equal(keys, rk) and np.array_equal(fr, np.asarray(rf, dtype=np.uint8))
        # interval points per key: the fusion rule looks at consecutive records of one hash, so a tie between two records of
        # the SAME hash cannot occur (same wpos and hash are de-duplicated): the lists must be identical
        assert np.array_equal(ko, ro)
        for f in ("pos", "seqId", "side", "hash"):
            if not np.array_equal(pts[f], rp[f]):
                bad = np.nonzero(pts[f] != rp[f])[0]
                i = int(bad[0])
                ki = int(np.searchsorted(ko, i, side="right") - 1)
                lo, hi = int(ko[ki]), int(ko[ki + 1])
                print(f"first {f} mismatch at point {i} ({len(bad)} in all), key {ki} = {int(keys[ki]):#x}, frequent {int(fr[ki])}")
                print("  device   :", [(int(p["seqId"]), int(p["pos"]), int(p["side"])) for p in pts[lo:hi]][:24])
                print("  reference:", [(int(p["seqId"]), int(p["pos"]), int(p["side"])) for p in rp[lo:hi]][:24])
                full = R.index()
                print("  reference minmers of that hash after the drop:", [(int(m["seqId"]), int(m["wpos"]), int(m["wpos_end"])) for m in full[full["hash"] == keys[ki]]][:24])
            assert np.array_equal(pts[f], rp[f]), f
        if expect_fixed is not None:
            assert (st["n_fixed_chunks"] > 0) == expect_fixed, st
        ctx.close()
        return st
    finally:
        R.close()


def build_and_compare_stored(d, args, expect_fixed):
    """the device index against the digests of the reference's index for the same command line"""
    from mashmap_b200 import capi

    want = golden_ref.get("sessions", golden_ref.key_of(args, d))
    k, seg, s, pi, _ = want["params"]
    kmer_pct = float(args[args.index("--kmerThreshold") + 1]) if "--kmerThreshold" in args else 0.001
    ctx = capi.Context(kmer_size=k, seg_length=seg, sketch_size=s)
    seqs = np.concatenate(d["genome"]).astype(np.uint8)
    offs = np.zeros(len(d["genome"]) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(c) for c in d["genome"]])
    st = ctx.index_build(seqs, offs, kmer_pct_threshold=kmer_pct, keep_lookup=True)
    print("device index:", st)
    mi, keys, ko, pts, fr = ctx.index_download()
    assert golden_ref.index_digests(mi, keys, ko, pts, fr, st["freq_threshold"]) == want["index"]
    if expect_fixed is not None:
        assert (st["n_fixed_chunks"] > 0) == expect_fixed, st
    ctx.close()
    return st


def test_index_random_genome(workdir, monkeypatch):
    d = datasets.make_random_set(workdir, tag="ixr")
    st = build_and_compare(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "4"], chunk=8192, monkeypatch=monkeypatch,
                           expect_fixed=False)
    assert st["n_chunks"] > 100


def test_index_panel_with_frequent_seeds(workdir, monkeypatch):
    d = datasets.make_panel_set(workdir, tag="ixp")
    build_and_compare(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "--kmerThreshold", "5", "-t", "4"], chunk=6000,
                      monkeypatch=monkeypatch)


def test_index_default_chunks_dense_sketch(workdir):
    d = datasets.make_big_random_set(workdir, tag="ixb", n_contigs=4, contig_len=1_000_000, n_reads=2)
    st = build_and_compare(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "95", "--dense", "-t", "8"], expect_fixed=False)
    assert st["n_chunks"] >= 80


@pytest.mark.parametrize("w,s,k", [(1000, 20, 19), (5000, 130, 19), (500, 10, 16), (2000, 64, 21)])
def test_index_degenerate_contigs(workdir, monkeypatch, w, s, k):
    """tandem repeats, N runs (also inside the first k-1 bases), low complexity, a palindrome, contigs shorter than a window
    and shorter than k: chunks whose record buffer overflows or whose warm-up state cannot be trusted are re-scanned exactly.
    These inputs are full of exact (wpos, wpos_end) ties, whose order -- and, through the adjacent de-duplication that
    follows the sort (commonFunc.hpp:563-568), even whose number -- the reference leaves to std::sort. So the device index is
    compared with the host run of the same window machine under the device's documented tie rule (emission order); that
    host run with std::sort instead is what tests/test_host_cpu.py pins to the reference record for record."""
    import test_host_cpu as t
    from mashmap_b200 import capi, hostlib

    cases = t._cases_for_index()
    genome = [v if isinstance(v, np.ndarray) else np.frombuffer(bytes(v), dtype=np.uint8).copy() for v in cases.values()]
    monkeypatch.setenv("MM_INDEX_CHUNK", str(max(1024, w // 2 * 3)))
    ctx = capi.Context(kmer_size=k, seg_length=w, sketch_size=s)
    seqs = np.concatenate(genome).astype(np.uint8)
    offs = np.zeros(len(genome) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(c) for c in genome])
    st = ctx.index_build(seqs, offs, kmer_pct_threshold=0.0, keep_lookup=True)
    print("device index:", st)
    assert st["n_fixed_chunks"] > 0 and st["freq_threshold"] == 2**31 - 1
    mi = ctx.index_download()[0]
    want = np.concatenate([hostlib.add_minmers(g, k, w, s, seq_id=i, stable_ties=True) for i, g in enumerate(genome)])
    assert len(mi) == len(want), (len(mi), len(want))
    for f in ("hash", "wpos", "wpos_end", "seqId", "strand"):
        assert np.array_equal(mi[f], want[f]), f
    # and against the reference itself wherever its order is defined: the records outside tie groups
    if not refh.available():
        ctx.close()
        return
    exact = np.concatenate([refh.add_minmers(g, k, w, s, seq_id=i) for i, g in enumerate(genome)])
    def untied(a):
        key = np.stack([a["seqId"].astype(np.int64), a["wpos"].astype(np.int64), a["wpos_end"].astype(np.int64)], axis=1)
        same_prev = np.zeros(len(a), bool); same_next = np.zeros(len(a), bool)
        same_prev[1:] = np.all(key[1:] == key[:-1], axis=1); same_next[:-1] = same_prev[1:]
        return a[~(same_prev | same_next)]
    a, b = untied(mi), untied(exact)
    same = len(a) == len(b) and all(np.array_equal(a[f], b[f]) for f in ("hash", "wpos", "wpos_end", "seqId", "strand"))
    # (a record next to a tie group can itself be kept or dropped by the de-duplication depending on the group's order, so
    # this is reported, not asserted)
    print(f"device {len(mi)} records / reference {len(exact)}; outside tie groups {len(a)} / {len(b)}, identical: {same}")
    ctx.close()
