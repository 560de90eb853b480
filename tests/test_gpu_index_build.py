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


# ---- small grids, many chains, rejected blocks ------------------------------------------------------------------------
# MM_INDEX_MACHINES caps the window-scan grid, so that each machine scans many chunks one after another in its own slab.
# A low-complexity block makes about two records per position, more than a chunk's record buffer (chunk/4 + s + 64)
# holds: every chunk with enough of it is rejected and re-scanned exactly.
LOW_COMPLEXITY = b"ACACACACACGTGTGTGTGT"


def _low_block(n):
    return np.frombuffer(LOW_COMPLEXITY * (n // len(LOW_COMPLEXITY)), np.uint8)


def _device_minmers(genome, k, w, s, monkeypatch, chunk, machines=None):
    from mashmap_b200 import capi

    monkeypatch.setenv("MM_INDEX_CHUNK", str(chunk))
    if machines is not None:
        monkeypatch.setenv("MM_INDEX_MACHINES", str(machines))
    ctx = capi.Context(kmer_size=k, seg_length=w, sketch_size=s)
    try:
        seqs = np.concatenate(genome).astype(np.uint8)
        offs = np.zeros(len(genome) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(c) for c in genome])
        st = ctx.index_build(seqs, offs, kmer_pct_threshold=0.0, keep_lookup=True)
        return st, ctx.index_download()[0]
    finally:
        ctx.close()


def _assert_host_minmers(mi, genome, k, w, s):
    """the device index against the host builder with the device's tie rule (see test_index_degenerate_contigs)"""
    from mashmap_b200 import hostlib

    want = np.concatenate([hostlib.add_minmers(g, k, w, s, seq_id=i, stable_ties=True) for i, g in enumerate(genome)])
    assert len(mi) == len(want), (len(mi), len(want))
    for f in ("hash", "wpos", "wpos_end", "seqId", "strand"):
        assert np.array_equal(mi[f], want[f]), f


def _touched_chunks(begin, end, k, chunk):
    """the chunks (of k-mer positions) whose k-mers read a base of [begin, end)"""
    return set(range(max(0, begin - k + 1) // chunk, (end - 1) // chunk + 1))


@pytest.mark.parametrize("case", ["random", "panel", "big"])
def test_index_many_chunks_per_machine(workdir, monkeypatch, case):
    """a grid of 128 machines over 1,024-position chunks: every machine scans many chunks in turn, reusing its slab"""
    monkeypatch.setenv("MM_INDEX_MACHINES", "128")
    if case == "random":
        d = datasets.make_random_set(workdir, tag="ixr")
        args = ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "4"]
    elif case == "panel":
        d = datasets.make_panel_set(workdir, tag="ixp")
        args = ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "--kmerThreshold", "5", "-t", "4"]
    else:
        d = datasets.make_big_random_set(workdir, tag="ixb", n_contigs=4, contig_len=1_000_000, n_reads=2)
        args = ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "95", "--dense", "-t", "8"]
    st = build_and_compare(d, args, chunk=1024, monkeypatch=monkeypatch, expect_fixed=False if case != "panel" else None)
    assert st["n_chunks"] >= 8 * 128, st  # at least eight chunks per machine (about thirty on the big set)


def test_index_more_chains_than_machines(monkeypatch):
    """240 contigs, each with a low-complexity block, on a grid of 128 machines. The first rejected chunk of a contig is
    decided in round 0 (all of the contig before it is good), so round 0 re-scans one chain per contig: 240 chains, more
    than the grid's slabs"""
    k, w, s, chunk = 16, 500, 10, 1024
    rng = np.random.default_rng(23)
    low = _low_block(800)
    genome = []
    for i in range(240):
        g = synth.random_sequence(4000 + 37 * (i % 50), rng)
        at = 1100 + 7 * (i % 100)
        g[at : at + len(low)] = low
        genome.append(g)
    st, mi = _device_minmers(genome, k, w, s, monkeypatch, chunk, machines=128)
    print("device index:", st)
    assert st["n_fixed_chunks"] >= len(genome), st
    _assert_host_minmers(mi, genome, k, w, s)


def test_index_one_rejected_block_rescans_only_its_chunks(monkeypatch):
    """a 1.1 Mbp contig of random sequence with one low-complexity block whose end sweeps the offsets 0 .. warm before a
    chunk boundary: only the chunks the block touches (and at most two after them) are re-scanned, not the rest of the
    contig, and the index is the host builder's"""
    k, w, s, chunk = 19, 1000, 20, 4096
    warm = w + 2 * k + 64  # the warm-up of mm_index_build.cu
    rng = np.random.default_rng(29)
    base = synth.random_sequence(1_100_000, rng)
    low = _low_block(3000)
    boundary = 40 * chunk
    n_chunks = (len(base) - k + 1 + chunk - 1) // chunk
    rounds = {}
    for end in sorted({0, 1, k - 1, k, w // 2, w - 1, w, w + 1, w + k, warm - 64, warm - 1, warm}):
        g = base.copy()
        e = boundary - end
        g[e - len(low) : e] = low
        st, mi = _device_minmers([g], k, w, s, monkeypatch, chunk)
        touched = _touched_chunks(e - len(low), e, k, chunk)
        print(f"block end {end} before a boundary: {len(touched)} chunks touched, {st['n_fixed_chunks']} re-scanned in "
              f"{st['fix_rounds']} rounds, of {n_chunks}")
        assert st["n_chunks"] == n_chunks
        assert 1 <= st["n_fixed_chunks"] <= len(touched) + 2, (end, st)
        _assert_host_minmers(mi, [g], k, w, s)
        rounds[end] = st["fix_rounds"]
    # One round at every offset: the chunk after the re-scanned block always matched the block's exact end state, so the
    # branch that extends a re-scanned chain is not reached here. It stays, since a chunk that does not match can only be
    # re-scanned as part of that chain: a new chain would have to start from a rejected chunk's untrusted warm-up state.
    # fix_rounds >= 2 is reached by separate rejected runs (test_index_many_rejected_blocks_in_one_contig).
    print("rounds by offset:", rounds)


def test_index_many_rejected_blocks_in_one_contig(monkeypatch):
    """300 low-complexity blocks 1, 2 and 3 chunks apart in one contig: one round per separate run of rejected chunks, each
    chain bounded by the chunks its block touches, and the index is the host builder's"""
    k, w, s, chunk = 19, 1000, 20, 4096
    rng = np.random.default_rng(31)
    low = _low_block(3000)
    starts, c = [], 2
    for i in range(300):
        starts.append(c * chunk + 200)
        c += 1 + i % 3
    g = synth.random_sequence((c + 2) * chunk, rng)
    allowed = set()
    for a in starts:
        g[a : a + len(low)] = low
        t = _touched_chunks(a, a + len(low), k, chunk)
        allowed |= t | {max(t) + 1}
    st, mi = _device_minmers([g], k, w, s, monkeypatch, chunk, machines=128)
    print("device index:", st, f"{len(allowed)} chunks touched or right after a block")
    assert len(starts) <= st["n_fixed_chunks"] <= len(allowed), st
    assert st["fix_rounds"] >= 2, st
    _assert_host_minmers(mi, [g], k, w, s)
