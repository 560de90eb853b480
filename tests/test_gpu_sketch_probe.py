"""The lookup-table probe of every query sketch hash happens inside the sketch kernels (K1): the fast kernel, the general
kernel (for the segments the fast kernel rejects, and for every segment under MM_SKETCH_TABLE=1) and the merge of a long
fragment's pieces each look up the hashes they write. Checked stage by stage against the oracle's restatement
(oracle/mm_oracle.cpp, pinned against the reference by test_oracle.py) on an index built on the device, in batches that
take every one of those paths, with frequent seeds in the index; and a sketch-only call on a context without an index."""
import numpy as np
import pytest

import golden_ref
import oracle_py
from conftest import have_gpu
from mashmap_b200 import synth

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not have_gpu(), reason="no GPU")]

K, SEG, S, PI = 19, 2000, 60, 0.85


def repeat_rich_genome(seed=71):
    """two random contigs; the second carries 200 copies of one 1.5 kb element and 40 of another, whose k-mers the index
    flags frequent"""
    rng = np.random.default_rng(seed)
    elements = [synth.random_sequence(1500, rng), synth.random_sequence(1200, rng)]
    parts = []
    for i in range(240):
        parts += [elements[0] if i % 6 else elements[1], synth.random_sequence(int(rng.integers(200, 600)), rng)]
    return [synth.random_sequence(300_000, rng), np.concatenate(parts)]


def mixed_reads(genome, seed=72):
    """reads drawn from the genome (some through the repeat), and reads the fast kernel hands over: a homopolymer run,
    a short tandem repeat, N-rich reads"""
    rng = np.random.default_rng(seed)
    reads, _ = synth.simulate_reads(genome, 24, 6000, 0.01, 0.06, seed=seed)
    reads = list(reads)
    base = reads[0].copy()
    homo = base.copy(); homo[500:4500] = ord("A")
    tandem = np.tile(synth.random_sequence(37, rng), 200)[:6000]
    nrich = reads[1].copy(); nrich[::50] = ord("N")
    nblock = reads[2].copy(); nblock[1000:3500] = ord("N")
    return reads + [homo, tandem, nrich, nblock]


def device_context(genome, kmer_pct_threshold=1.0):
    """a context holding an index built on the device, and the oracle on the same index. The frequent-seed cut is
    1 % of the distinct keys (the CLI's default, 0.001 %, flags nothing in an index this small)"""
    from mashmap_b200 import capi, hostlib

    ctx = capi.Context(kmer_size=K, seg_length=SEG, sketch_size=S)
    offs = np.zeros(len(genome) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(c) for c in genome])
    ctx.index_build(np.concatenate(genome), offs, kmer_pct_threshold=kmer_pct_threshold, keep_lookup=True)
    idx, keys, offs_, pts, freq = ctx.index_download()
    ctx.tables_upload(hostlib.sketch_cutoffs(S, K), hostlib.min_hits_table(S, K, PI))
    O = oracle_py.Oracle(K, SEG, S, PI)
    O.set_index(idx, keys, offs_, pts, freq, [len(c) for c in genome])
    return ctx, O, freq


def segments(seqs_and_counters):
    from mashmap_b200 import capi

    segs = np.zeros(len(seqs_and_counters), dtype=capi.segment_dtype)
    off = 0
    for i, (q, counter) in enumerate(seqs_and_counters):
        segs[i]["offset"] = off; segs[i]["length"] = len(q); segs[i]["seq_counter"] = counter
        segs[i]["name_id"] = -1; segs[i]["ref_group"] = -1
        off += len(q)
    return np.concatenate([q for q, _ in seqs_and_counters]), segs


def compare_with_oracle(O, frags, seg_res, cands, loci):
    """per fragment: sketch size after frequent-seed removal, interval points, L1 candidates, L2 loci"""
    bad = []
    for i, (q, counter) in enumerate(frags):
        exp = O.map_fragment(q, seq_counter=counter, full_len=len(q))
        sr = seg_res[i]
        if sr["sketch_size"] != exp["sketch_size"] or sr["n_points"] != exp["n_points"]:
            bad.append((i, "sketch_size / n_points", int(sr["sketch_size"]), exp["sketch_size"], int(sr["n_points"]), exp["n_points"]))
            continue
        c = cands[sr["first_candidate"] : sr["first_candidate"] + sr["n_candidates"]]
        if len(c) != len(exp["l1"]) or not all(np.array_equal(c[f], exp["l1"][f])
                                               for f in ("seqId", "rangeStartPos", "rangeEndPos", "intersectionSize")):
            bad.append((i, "l1"))
            continue
        for ci in range(len(c)):
            dl = loci[c[ci]["first_locus"] : c[ci]["first_locus"] + c[ci]["n_loci"]]
            el = exp["l2"][exp["l2_cand"] == ci]
            if len(dl) != len(el) or not all(np.array_equal(dl[f], el[f]) for f in el.dtype.names):
                bad.append((i, f"l2 cand {ci}"))
    return bad


@pytest.mark.parametrize("mode", ["fast+general", "general-only"])
def test_mixed_batch_with_rejects_and_frequent_seeds(mode, monkeypatch):
    """fast-kernel segments next to the ones it rejects to the general kernel, hashes flagged frequent in the index"""
    if mode == "general-only":
        monkeypatch.setenv("MM_SKETCH_TABLE", "1")
    genome = repeat_rich_genome()
    ctx, O, freq = device_context(genome)
    try:
        reads = mixed_reads(genome)
        lens = [len(r) for r in reads]
        ridx, start, length = synth.split_segments(lens, SEG, K)
        frags = [(reads[r][s : s + n], int(r)) for r, s, n in zip(ridx, start, length)]
        bases, segs = segments(frags)
        seg_res, cands, loci = ctx.map_segments(bases, segs)
        bad = compare_with_oracle(O, frags, seg_res, cands, loci)
        print("mismatches:", bad[:10], "diag:", ctx.diag())
        assert not bad
        assert int(np.asarray(freq).sum()) > 0
        assert int((seg_res["sketch_raw_count"] - seg_res["sketch_size"]).sum()) > 0, "no frequent seed reached a sketch"
        assert seg_res["n_candidates"].sum() > 0
        if mode == "fast+general":
            assert ctx.diag()["sketch_general_segments"] > 0, "no segment took the general kernel"
    finally:
        O.close()
        ctx.close()


def test_long_fragments_next_to_segments():
    """--noSplit: fragments longer than a segment (sketched as pieces and merged) between ordinary segments"""
    genome = repeat_rich_genome(seed=81)
    ctx, O, _ = device_context(genome)
    try:
        reads, _ = synth.simulate_reads(genome, 10, 9000, 0.01, 0.05, seed=82)
        frags = []
        for i, r in enumerate(reads):
            frags.append((r if i % 2 == 0 else r[:SEG], i))
        bases, segs = segments(frags)
        seg_res, cands, loci = ctx.map_segments(bases, segs)
        bad = compare_with_oracle(O, frags, seg_res, cands, loci)
        print("mismatches:", bad[:10], "diag:", ctx.diag())
        assert not bad
        assert ctx.diag()["long_fragments"] == sum(len(q) > SEG for q, _ in frags)
        assert seg_res["n_candidates"][[len(q) > SEG for q, _ in frags]].sum() > 0
    finally:
        O.close()
        ctx.close()


def test_sketch_only_without_an_index():
    """mm_sketch_segments needs no index: the kernels skip the probe"""
    from mashmap_b200 import capi

    genome = repeat_rich_genome()
    seqs = mixed_reads(genome)[-6:]
    ctx = capi.Context(kmer_size=K, seg_length=SEG, sketch_size=S)
    frags = [(q[:SEG], i) for i, q in enumerate(seqs)] + [(seqs[0], len(seqs))]
    bases, segs = segments(frags)
    out, cnt = ctx.sketch_segments(bases, segs)
    for i, (q, counter) in enumerate(frags):
        want = oracle_py.sketch_sequence(q, K, S, seq_id=counter)
        assert golden_ref.sketch_digest(out[i], cnt[i]) == golden_ref.sketch_digest(want), i
    assert ctx.diag()["sketch_general_segments"] > 0
    ctx.close()
