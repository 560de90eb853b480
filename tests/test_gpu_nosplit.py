"""Queries mapped as ONE fragment longer than a segment (--noSplit, windowLen = length - segLength > 0) on the GPU, through
the C ABI and the CLI, bit for bit against the unmodified reference (oracle/_ref where it is built, otherwise its results
stored by tests/golden/make_nosplit_golden.py):
  K1  the device cuts such a fragment into pieces, sketches them with the ordinary sketch kernels and merges them: equal
      to CommonFunc::sketchSequence over the whole fragment (and to the oracle's restatement of it);
  K2 / K3  k_l1_long / k_l2_long: sketch, interval points, L1 candidates and L2 loci per candidate of every whole query
      equal mapSingleQueryFrag's, with the fast and the general kernels of the other fragments;
  CLI  mashmap-b200 --noSplit prints the reference's PAF."""
import os
import subprocess

import numpy as np
import pytest

import golden_ref
import nosplit_data as ND
import oracle_py
import refh
import test_gpu_stages as T
from conftest import have_gpu

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not have_gpu(), reason="no GPU")]


def segments_of(seqs):
    from mashmap_b200 import capi

    segs = np.zeros(len(seqs), dtype=capi.segment_dtype)
    off = 0
    for i, q in enumerate(seqs):
        segs[i]["offset"] = off; segs[i]["length"] = len(q); segs[i]["seq_counter"] = i; segs[i]["name_id"] = -1
        segs[i]["ref_group"] = -1
        off += len(q)
    return np.concatenate(seqs), segs


def reference_digests(key, seqs, k, s):
    if refh.available():
        got = [golden_ref.sketch_digest(refh.sketch_sequence(q, k, s, seq_id=i)) for i, q in enumerate(seqs)]
        ND.check_stored("sketch_long", key, got)
        return got
    return ND.get("sketch_long", key)


@pytest.mark.parametrize("mode", ["fast+general", "general-only"])
@pytest.mark.parametrize("k,s", ND.SKETCH_CASES)
def test_long_fragment_sketch_equals_reference(k, s, mode, monkeypatch):
    from mashmap_b200 import capi

    if mode == "general-only":
        monkeypatch.setenv("MM_SKETCH_TABLE", "1")
    seqs = ND.long_sequences(k)
    ctx = capi.Context(kmer_size=k, seg_length=ND.SEG, sketch_size=s)
    bases, segs = segments_of(seqs)
    out, cnt = ctx.sketch_segments(bases, segs)
    want = reference_digests(f"k{k} s{s}", seqs, k, s)
    bad = []
    for i, q in enumerate(seqs):
        dev = out[i][: cnt[i]]
        orc = oracle_py.sketch_sequence(q, k, s, seq_id=i)
        if golden_ref.sketch_digest(dev) != want[i]:
            bad.append((i, len(q), "reference"))
        if golden_ref.sketch_digest(dev) != golden_ref.sketch_digest(orc) or not np.all(dev["seqId"] == i):
            bad.append((i, len(q), "oracle"))
    print("mismatches:", bad)
    assert not bad
    assert ctx.diag()["long_fragments"] == sum(len(q) > ND.SEG for q in seqs)
    ctx.close()


def test_short_segments_unchanged_next_to_long_fragments():
    """a batch of ordinary segments gives the same sketches with and without long fragments between them"""
    from mashmap_b200 import capi

    k, s = 19, 100
    short = ND.short_sequences()
    longs = ND.long_sequences(k)[:4]
    ctx = capi.Context(kmer_size=k, seg_length=ND.SEG, sketch_size=s)
    b0, s0 = segments_of(short)
    o0, c0 = ctx.sketch_segments(b0, s0)
    mixed = [longs[0], short[0], longs[1], short[1], short[2], longs[2], longs[3], short[3]]
    where = [1, 3, 4, 7]
    b1, s1 = segments_of(mixed)
    o1, c1 = ctx.sketch_segments(b1, s1)
    for j, i in enumerate(where):
        assert c1[i] == c0[j]
        a, b = o1[i][: c1[i]].copy(), o0[j][: c0[j]].copy()
        a["seqId"] = 0; b["seqId"] = 0
        assert a.tobytes() == b.tobytes(), (i, j)
    for i in (0, 2, 5, 6):
        assert golden_ref.sketch_digest(o1[i], c1[i]) == golden_ref.sketch_digest(oracle_py.sketch_sequence(mixed[i], k, s, seq_id=i))
    ctx.close()


def test_fragment_at_the_length_limit_is_refused():
    """2^30 k-mer positions: the reference's (len - k + 1) * 2 overflows an int (computeMap.hpp:831)"""
    from mashmap_b200 import capi

    k = 19
    ctx = capi.Context(kmer_size=k, seg_length=ND.SEG, sketch_size=100)
    segs = np.zeros(1, dtype=capi.segment_dtype)
    segs[0]["length"] = (1 << 30) + k - 1
    with pytest.raises(capi.MashmapError, match="2\\^30"):
        ctx.sketch_segments(np.zeros(16, np.uint8), segs)
    ctx.close()


@pytest.fixture(scope="module")
def data_sets(workdir):
    make, made = ND.datasets_by_name(workdir), {}

    def get(name):
        if name not in made:
            made[name] = make[name]()
        return made[name]
    return get


def whole_query_segments(d, k):
    from mashmap_b200 import capi

    ridx, lens = ND.whole_reads(d, k)
    offs = np.zeros(len(d["reads"]) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(r) for r in d["reads"]])
    segs = np.zeros(len(ridx), dtype=capi.segment_dtype)
    segs["offset"] = offs[ridx]
    segs["length"] = lens
    segs["seq_counter"] = ridx
    segs["name_id"] = -1
    segs["ref_group"] = -1
    return np.concatenate(d["reads"]).astype(np.uint8), segs, ridx, lens


def reference_fragment_digests(R, d, ridx, lens):
    if isinstance(R, refh.RefSession):
        got = [golden_ref.reference_fragment_digest(R.map_fragment(d["rnames"][i], d["reads"][i], full_len=int(n), seq_counter=int(i)))
               for i, n in zip(ridx, lens)]
        ND.check_stored("fragments", R.key, got)
        return got
    return ND.get("fragments", R.key)


def map_whole_queries(R, bases, segs, fetched=None):
    """(digests per fragment, seg_res, ctx diag) through mm_map_segments, checked equal to the resident path; the resident
    path's candidates and loci are appended to `fetched` when it is a list"""
    from mashmap_b200 import capi

    ctx = capi.Context(kmer_size=R.p.kmerSize, seg_length=R.p.segLength, sketch_size=R.p.sketchSize,
                       stage1_topani_filter=bool(R.p.stage1_topANI_filter))
    T.upload_reference_index(ctx, R)
    seg_res, cands, loci = ctx.map_segments(bases, segs)
    ctx.batch_upload(bases, segs)
    ctx.map_resident()
    seg_res2, cands2, loci2 = ctx.batch_fetch()
    sk, cnt = ctx.batch_fetch_sketch()
    got = [T.device_fragment_digest(i, seg_res2, cands2, loci2, sk, cnt) for i in range(len(segs))]
    first = [T.device_fragment_digest(i, seg_res, cands, loci, sk, cnt) for i in range(len(segs))]
    assert got == first, "mm_map_segments and the resident path differ"
    print("stage ms", ctx.stage_ms(), "diag", ctx.diag(), "candidates", len(cands2), "loci", len(loci2))
    dg = ctx.diag()
    ctx.close()
    if fetched is not None:
        fetched += [cands2, loci2]
    return got, seg_res2, dg


@pytest.mark.parametrize("which,opts", ND.STAGE_RUNS)
def test_whole_query_stages_equal_reference(data_sets, which, opts, kernel_paths):
    """every query of the data set as one fragment: sketch, n_points, L1 candidates, L2 loci per candidate"""
    d = data_sets(which)
    R = T.open_session(["-r", d["ref"], "-q", d["qry"]] + opts, d)
    try:
        bases, segs, ridx, lens = whole_query_segments(d, R.p.kmerSize)
        assert (lens > R.p.segLength).any()
        want = reference_fragment_digests(R, d, ridx, lens)
        got, seg_res, dg = map_whole_queries(R, bases, segs)
        bad = [(int(ridx[i]), int(lens[i])) for i in range(len(segs)) if got[i] != want[i]]
        print(f"{which} {opts}: {len(segs)} queries, {int((lens > R.p.segLength).sum())} longer than a segment, "
              f"candidates {int(seg_res['n_candidates'].sum())}, mismatches {bad}")
        assert not bad
        assert dg["long_fragments"] >= int((lens > R.p.segLength).sum())
        assert seg_res["n_candidates"][lens > R.p.segLength].sum() > 0
    finally:
        R.close()


@pytest.fixture(params=["fast-paths", "general-kernels"])
def kernel_paths(request, monkeypatch):
    """the fragments next to the long ones on the fast kernels (default) or on the general kernels alone"""
    if request.param == "general-kernels":
        monkeypatch.setenv("MM_SKETCH_TABLE", "1")
        monkeypatch.setenv("MM_L1_CTA", "1")
        monkeypatch.setenv("MM_L2_GENERAL", "1")
    return request.param


def test_segments_unchanged_next_to_long_fragments(data_sets):
    """the split fragments of a batch give the same results with and without whole queries between them"""
    d = data_sets("random")
    R = T.open_session(["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "4"], d)
    try:
        from mashmap_b200 import capi

        bases, segs, ridx, start, length = T.build_segments(d, R.p.segLength, R.p.kmerSize)
        alone, _, _ = map_whole_queries(R, bases, segs)
        _, whole, _, _ = whole_query_segments(d, R.p.kmerSize)
        mixed = np.zeros(len(segs) + len(whole), dtype=capi.segment_dtype)
        is_split = np.ones(len(mixed), dtype=bool)
        is_split[1::3][: len(whole)] = False
        mixed[~is_split] = whole[: int((~is_split).sum())]
        mixed[is_split] = segs
        got, _, dg = map_whole_queries(R, bases, mixed)
        assert [g for g, s in zip(got, is_split) if s] == alone
        assert dg["long_fragments"] > 0
    finally:
        R.close()


def run_cli(cmd):
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 0, (cmd, p.stderr[-2000:])
    return p.stderr


def paf_rows(path):
    return [line.rstrip("\n").split("\t") for line in open(path)]


@pytest.mark.parametrize("which,opts", ND.CLI_RUNS)
def test_cli_nosplit_prints_reference_paf(data_sets, workdir, which, opts):
    from mashmap_b200 import hostlib

    d = data_sets(which)
    name = ND.cli_name(which, opts)
    stored = os.path.join(ND.PAF_DIR, name + ".paf")
    if os.path.exists(refh.REF_BIN):
        ref_out = os.path.join(workdir, "ref_ns_" + name + ".paf")
        run_cli([refh.REF_BIN, "-r", d["ref"], "-q", d["qry"], "-t", "8", "--noSplit", "-o", ref_out] + opts)
        assert open(ref_out).read() == open(stored).read(), f"{stored} is stale"
    got_out = os.path.join(workdir, "got_ns_" + name + ".paf")
    run_cli([hostlib.CLI_PATH, "-r", d["ref"], "-q", d["qry"], "-t", "8", "--noSplit", "-o", got_out] + opts)
    ref, got = paf_rows(stored), paf_rows(got_out)
    print(f"{which} {opts}: reference {len(ref)} lines, ours {len(got)}")
    assert len(ref) > 0
    assert [r[:12] for r in ref] == [g[:12] for g in got]
    for r, g in zip(ref, got):
        assert abs(float(r[12].split(":")[2]) - float(g[12].split(":")[2])) <= 1e-4, (r, g)
        assert abs(float(r[13].split(":")[2]) - float(g[13].split(":")[2])) <= 1e-4 * max(1.0, abs(float(r[13].split(":")[2])))
    # one batch smaller than a query: the output does not change
    small_out = os.path.join(workdir, "got_ns_small_" + name + ".paf")
    run_cli([hostlib.CLI_PATH, "-r", d["ref"], "-q", d["qry"], "-t", "8", "--noSplit", "--batchBases", "20000", "-o", small_out] + opts)
    assert open(small_out).read() == open(got_out).read()
