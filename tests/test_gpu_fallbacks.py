"""The mapping context's regrow paths against the reference: a candidate or locus buffer that is too small is grown and the
stage rerun, and the result must be the one a large enough buffer gives. MM_CAND_ELEMS and MM_LOCI_ELEMS shrink the
buffers a fresh context starts with, so that the small test batches take these paths; every row asserts the counter
that shows its path ran."""
import numpy as np
import pytest

import fallback_data as FD
import nosplit_data as ND
from conftest import have_gpu
from test_gpu_stages import (build_segments, kernel_paths, open_session, panel_set, random_set, repeat_set,  # noqa: F401
                             run_stage_parity, upload_reference_index)

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not have_gpu(), reason="no GPU")]


def _args(d, *extra):
    return ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", *extra, "-t", "4"]


@pytest.mark.parametrize("case", ["random", "panel", "repeat"])
def test_candidate_regrow(random_set, panel_set, repeat_set, kernel_paths, monkeypatch, case):
    """a candidate buffer of one element: K2 reports how many it needs, the host grows the buffer and reruns K1 and K2"""
    monkeypatch.setenv("MM_CAND_ELEMS", "1")
    d = {"random": random_set, "panel": panel_set, "repeat": repeat_set}[case]
    extra = ("--noHgFilter",) if case == "repeat" else ()
    bad = run_stage_parity(d, _args(d, *extra), 5000, expect_diag=("cand_regrow",))
    assert not bad


WHOLE_RUNS = [r for r in ND.STAGE_RUNS if r[0] in ("random", "panel") or "--noHgFilter" in r[1]]


@pytest.mark.parametrize("which,opts", WHOLE_RUNS)
def test_candidate_regrow_whole_queries(workdir, kernel_paths, monkeypatch, which, opts):
    """--noSplit: every query one fragment (k_l1_long / k_l2_long for those longer than a segment) with a candidate buffer of
    one element; the call that regrew equals the resident call, and both the reference"""
    import test_gpu_nosplit as NS

    monkeypatch.setenv("MM_CAND_ELEMS", "1")
    d = ND.datasets_by_name(workdir)[which]()
    R = open_session(["-r", d["ref"], "-q", d["qry"]] + opts, d)
    try:
        bases, segs, ridx, lens = NS.whole_query_segments(d, R.p.kmerSize)
        want = NS.reference_fragment_digests(R, d, ridx, lens)
        got, _, dg = NS.map_whole_queries(R, bases, segs)
        print(which, opts, "diag", dg)
        assert got == want
        assert dg["long_fragments"] > 0 and dg["cand_regrow"] > 0, dg
    finally:
        R.close()


def test_locus_regrow(repeat_set, kernel_paths, monkeypatch):
    """no locus room beyond the stream kernel's fixed slots: the loci of the candidates with more than two of them overflow.
    On the fast paths the stream driver regrows (and reruns prep, order and scan); under MM_L2_GENERAL=1 the general
    driver does"""
    monkeypatch.setenv("MM_LOCI_ELEMS", "0")
    d = repeat_set
    bad = run_stage_parity(d, _args(d, "--noHgFilter"), 5000, expect_diag=("l2_loci_regrow",))
    assert not bad


def test_every_buffer_at_its_smallest(repeat_set, kernel_paths, monkeypatch):
    """the candidate, locus and L1 point-pool buffers all at their smallest at once"""
    monkeypatch.setenv("MM_CAND_ELEMS", "1")
    monkeypatch.setenv("MM_LOCI_ELEMS", "0")
    monkeypatch.setenv("MM_L1_POOL_ELEMS", "4096")
    d = repeat_set
    bad = run_stage_parity(d, _args(d, "--noHgFilter"), 5000, expect_diag=("cand_regrow", "l2_loci_regrow", "l1_pool_regrow"))
    assert not bad


def test_long_driver_regrows_and_keeps_the_loci_before_it(random_set, monkeypatch):
    """k_l2_long appends the loci of whole queries after those of the split fragments of its batch. With no locus room
    beyond the stream kernel's fixed slots, and split fragments that fit those slots (random sequence: one or two loci
    each), the stream driver does not regrow and the long driver overflows: the buffer must grow keeping the loci before
    it. The split fragments of the mixed batch equal the batch without whole queries and the reference, and the mixed
    batch regrows where the split one does not. (On a tandem set the stream driver regrows first, with room to spare for
    the whole queries.)"""
    import golden_ref
    import refh
    import test_gpu_nosplit as NS
    from mashmap_b200 import capi

    monkeypatch.setenv("MM_LOCI_ELEMS", "0")
    d = random_set
    R = open_session(_args(d), d)
    try:
        bases, segs, ridx, start, length = build_segments(d, R.p.segLength, R.p.kmerSize)
        alone, _, dg_alone = NS.map_whole_queries(R, bases, segs)
        if isinstance(R, refh.RefSession):
            want = [golden_ref.reference_fragment_digest(R.map_fragment(d["rnames"][ridx[i]], d["reads"][ridx[i]][start[i] : start[i] + length[i]],
                                                                        full_len=len(d["reads"][ridx[i]]), seq_counter=int(ridx[i])))
                    for i in range(len(segs))]
        else:
            want = golden_ref.get("fragments", R.key)
        assert alone == want
        _, whole, _, _ = NS.whole_query_segments(d, R.p.kmerSize)
        whole = whole[whole["length"] > R.p.segLength][: len(segs) // 2]  # fragments for k_l2_long, between the split ones
        mixed = np.zeros(len(segs) + len(whole), dtype=capi.segment_dtype)
        is_split = np.ones(len(mixed), dtype=bool)
        is_split[1::3][: len(whole)] = False
        mixed[~is_split] = whole
        mixed[is_split] = segs
        got, _, dg_mixed = NS.map_whole_queries(R, bases, mixed)
        print("split only:", dg_alone, "mixed:", dg_mixed)
        assert [g for g, s in zip(got, is_split) if s] == alone
        assert dg_mixed["long_fragments"] > 0
        assert dg_mixed["l2_loci_regrow"] > dg_alone["l2_loci_regrow"], (dg_alone, dg_mixed)
    finally:
        R.close()


@pytest.mark.parametrize("copies", FD.TANDEM_COPIES)
def test_more_loci_than_the_staging_area(workdir, kernel_paths, copies):
    """a tandem array of 16, 17 and 24 exact copies: one candidate spans it and L2 finds a locus per copy. Beyond
    L2_STAGE_LOCI = 16 loci the general kernel runs its scan a second time, writing straight to the locus buffer; the
    stages must be the reference's, so the reference found as many"""
    d = FD.tandem_set(workdir, copies)
    most = []

    def check(seg_res, cands, loci):
        most.append(int(cands["n_loci"].max()))

    bad = run_stage_parity(d, FD.tandem_args(d), 5000, check=check)
    print("most loci of one candidate:", most)
    assert not bad
    if copies > 16:
        assert most[0] > 16


@pytest.mark.parametrize("copies", FD.TANDEM_COPIES)
def test_more_loci_than_the_staging_area_whole_queries(workdir, kernel_paths, copies):
    """the same tandem arrays under --noSplit: k_l2_long runs its own second scan beyond L2_STAGE_LOCI loci"""
    import test_gpu_nosplit as NS

    d = FD.tandem_set(workdir, copies)
    R = open_session(FD.tandem_args(d), d)
    try:
        bases, segs, ridx, lens = NS.whole_query_segments(d, R.p.kmerSize)
        want = NS.reference_fragment_digests(R, d, ridx, lens)
        fetched = []
        got, _, dg = NS.map_whole_queries(R, bases, segs, fetched)
        cands = fetched[0]
        most = int(cands["n_loci"].max())
        print("most loci of one candidate:", most, "diag", dg)
        assert got == want
        assert dg["long_fragments"] > 0
        if copies > 16:
            assert most > 16
    finally:
        R.close()


def _map(ctx, bases, segs):
    ctx.batch_upload(bases, segs)
    ctx.map_resident()
    return ctx.batch_fetch()


def _same(a, b):
    """each segment's results, candidates and their loci (where a segment's candidates land in the array depends on the
    order the device's blocks ran)"""
    from test_gpu_shards import per_segment

    assert per_segment(*a) == per_segment(*b)


def test_context_reuse_after_regrow(repeat_set, random_set, monkeypatch):
    """one context maps a batch that regrew, then a different batch, then the first batch again: each result equals a fresh
    context's, and the repeat finds its buffers large enough (no regrow counter moves)"""
    from mashmap_b200 import capi

    monkeypatch.setenv("MM_CAND_ELEMS", "1")
    monkeypatch.setenv("MM_LOCI_ELEMS", "0")
    monkeypatch.setenv("MM_L1_POOL_ELEMS", "4096")
    d = repeat_set
    R = open_session(_args(d, "--noHgFilter"), d)
    try:
        def fresh():
            ctx = capi.Context(kmer_size=R.p.kmerSize, seg_length=R.p.segLength, sketch_size=R.p.sketchSize,
                               stage1_topani_filter=bool(R.p.stage1_topANI_filter))
            upload_reference_index(ctx, R)
            return ctx

        a = build_segments(d, R.p.segLength, R.p.kmerSize)
        b = build_segments(random_set, R.p.segLength, R.p.kmerSize)  # other reads against the same index
        want = {}
        for name, (bases, segs, *_) in (("a", a), ("b", b)):
            ctx = fresh()
            want[name] = _map(ctx, bases, segs)
            ctx.close()
        ctx = fresh()
        _same(_map(ctx, a[0], a[1]), want["a"])
        dg1 = ctx.diag()
        print("after the first batch:", dg1)
        assert dg1["cand_regrow"] > 0 and dg1["l2_loci_regrow"] > 0 and dg1["l1_pool_regrow"] > 0, dg1
        _same(_map(ctx, b[0], b[1]), want["b"])
        dg2 = ctx.diag()
        _same(_map(ctx, a[0], a[1]), want["a"])
        dg3 = ctx.diag()
        print("after the second and third batch:", dg2, dg3)
        for name in ("cand_regrow", "l2_loci_regrow", "l1_pool_regrow"):
            assert dg3[name] == dg2[name], (name, dg2, dg3)
        ctx.close()
    finally:
        R.close()


@pytest.mark.parametrize("which,hg,whole,n", [("random", True, False, 2), ("random", False, False, 3), ("panel", True, True, 2),
                                              ("panel", False, True, 3)])
def test_sharded_phase_two_retry(workdir, kernel_paths, monkeypatch, which, hg, whole, n):
    """each shard maps with the best over all shards (phase 2), which skips K1 on its first attempt. A candidate buffer of
    one element makes that attempt overflow, so the retry reruns K1 from the bases; the merged stages must still equal the
    unsharded context's. Phase 1 emits no candidates, so a candidate regrow on a shard is phase 2's retry"""
    from test_gpu_shards import compare_sharded

    monkeypatch.setenv("MM_CAND_ELEMS", "1")
    monkeypatch.setenv("MM_L1_POOL_ELEMS", "4096")
    diags = compare_sharded(workdir, which, hg, whole, n)
    print("shard diagnostics:", diags)
    assert all(dg["cand_regrow"] > 0 for dg in diags), diags


HOOKS = {"MM_CAND_ELEMS": "1", "MM_LOCI_ELEMS": "0", "MM_L1_POOL_ELEMS": "4096", "MM_INDEX_MACHINES": "128", "MM_INDEX_CHUNK": "1024"}
CLI_ARGS = [[], ["--noSplit"], ["-f", "one-to-one"], ["--indexShards", "2"], ["--subBatchBases", "20000"]]


@pytest.mark.parametrize("args", CLI_ARGS, ids=lambda a: " ".join(a) or "default")
@pytest.mark.parametrize("which", ["repeat24", "random"])
def test_cli_paf_unchanged_with_every_buffer_at_its_smallest(workdir, which, args):
    """the CLI with every capacity hook at its smallest (a CLI process inherits them) writes the PAF it writes without them"""
    import os
    import re
    import subprocess

    import datasets
    from mashmap_b200 import hostlib

    if which == "repeat24":
        d = datasets.make_repeat_set(workdir, tag="rep24", tandem_copies=24)
        base = ["-s", "5000", "--pi", "85", "--noHgFilter"]
    else:
        d = datasets.make_random_set(workdir, tag="cli")
        base = ["-s", "5000", "--pi", "85"]
    tag = "_".join(a.strip("-") for a in args)
    outs = []
    for hooks in ({}, HOOKS):
        o = os.path.join(workdir, f"hooks{len(hooks)}_{which}_{tag}.paf")
        env = {k: v for k, v in os.environ.items() if k not in HOOKS}
        env.update(hooks)
        env["MM_TRACE"] = "1"  # one stderr line per part of a batch, naming the lane that mapped it
        p = subprocess.run([hostlib.CLI_PATH, "-r", d["ref"], "-q", d["qry"], "-t", "6", "-o", o] + base + args, env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        assert p.returncode == 0, p.stderr[-3000:]
        outs.append(open(o, "rb").read())
        lanes = set(re.findall(r"^\[trace\] lane (\d+) ", p.stderr, re.M))
        if "--subBatchBases" in args:
            assert len(lanes) >= 2, lanes  # the batch was cut into parts that several lanes mapped
    assert len(outs[0]) > 0
    assert outs[1] == outs[0]
