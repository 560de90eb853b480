"""GPU parity, stage by stage, through the C ABI, against the UNMODIFIED reference (oracle/_ref harness):
K1 sketch == CommonFunc::sketchSequence, K2 candidates == doL1Mapping, K3 loci == computeL2MappedRegions.
Bit-exact (integer work). Where the reference is not built, against its results stored in tests/golden (golden_ref.py)."""
import numpy as np
import pytest

import datasets
import golden_ref
import refh
from conftest import have_gpu
from mashmap_b200 import synth

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not have_gpu(), reason="no GPU")]


def open_session(args, d):
    """the reference's Sketch + Map for a command line, or, without the reference, the product's host index checked
    against the reference's stored digests"""
    key = golden_ref.key_of(args, d)
    if refh.available():
        R = refh.RefSession(args)
        golden_ref.check_stored("sessions", key, golden_ref.session_digests(R))
    else:
        R = golden_ref.ProductSession(args)
        assert golden_ref.session_digests(R) == golden_ref.get("sessions", key)
        R.contig_len = np.array([len(c) for c in d["genome"]], dtype=np.int32)
        R.contig_names = list(d["names"])
    R.key = key
    return R


def reference_sketch_digests(section, key, seqs, k, s, seq_ids):
    """per sequence: the digest of the reference's sketchSequence (computed, or stored)"""
    if refh.available():
        got = [golden_ref.sketch_digest(refh.sketch_sequence(q, k, s, seq_id=i)) for q, i in zip(seqs, seq_ids)]
        golden_ref.check_stored(section, key, got)
        return got
    return golden_ref.get(section, key)


def build_segments(d, seg_length, k, name_ids=None):
    from mashmap_b200 import capi

    lens = [len(r) for r in d["reads"]]
    ridx, start, length = synth.split_segments(lens, seg_length, k)
    offs = np.zeros(len(lens) + 1, dtype=np.int64)
    offs[1:] = np.cumsum(lens)
    bases = np.concatenate(d["reads"]).astype(np.uint8)
    segs = np.zeros(len(ridx), dtype=capi.segment_dtype)
    segs["offset"] = offs[ridx] + start
    segs["length"] = length
    segs["seq_counter"] = ridx
    segs["name_id"] = -1 if name_ids is None else np.asarray(name_ids)[ridx]
    segs["ref_group"] = -1
    return bases, segs, ridx, start, length


def upload_reference_index(ctx, R):
    idx = R.index()
    keys, offs, pts, fr = R.lookup()
    ctx.index_upload(idx, keys, offs, pts, fr, R.contig_len)
    ctx.tables_upload(R.cutoffs(), R.min_hits_table())


def device_fragment_digest(i, seg_res, cands, loci, dev_sketch, dev_count):
    sr = seg_res[i]
    c = cands[sr["first_candidate"] : sr["first_candidate"] + sr["n_candidates"]]
    l2 = [loci[x["first_locus"] : x["first_locus"] + x["n_loci"]] for x in c]
    return golden_ref.fragment_digest(dev_sketch[i][: dev_count[i]], int(sr["sketch_size"]), int(sr["n_points"]), c, l2)


def compare_stages(ctx, R, d, ridx, start, length, seg_res, cands, loci, dev_sketch, dev_count, max_report=10, diag=None):
    bad = []
    n_cmp = 0
    if not isinstance(R, refh.RefSession):  # the reference's stored per-fragment digests
        want = golden_ref.get("fragments", R.key)
        assert len(want) == len(ridx)
        for i in range(len(ridx)):
            if device_fragment_digest(i, seg_res, cands, loci, dev_sketch, dev_count) != want[i]:
                bad.append((i, "fragment digest"))
        n_cmp = len(cands)
        for b in bad[:max_report]:
            print("MISMATCH", b)
        print(f"segments={len(ridx)} candidates={n_cmp} mismatches={len(bad)} (stored reference digests)")
        return bad
    ref_digests = []
    for i in range(len(ridx)):
        r = d["reads"][ridx[i]]
        seg = r[start[i] : start[i] + length[i]]
        o = R.map_fragment(d["rnames"][ridx[i]], seg, full_len=len(r), seq_counter=int(ridx[i]))
        ref_digests.append(golden_ref.reference_fragment_digest(o))
        sr = seg_res[i]
        # sketch after frequent-seed removal
        rs = o["sketch"]
        ds = dev_sketch[i][: dev_count[i]]
        if len(rs) != len(ds) or not (np.array_equal(rs["hash"], ds["hash"]) and np.array_equal(rs["wpos"], ds["wpos"])
                                      and np.array_equal(rs["wpos_end"], ds["wpos_end"])
                                      and np.array_equal(rs["strand"], ds["strand"])):
            bad.append((i, "sketch", len(rs), len(ds)))
            continue
        if sr["sketch_size"] != len(rs):
            bad.append((i, "sketch_size", len(rs), int(sr["sketch_size"])))
        if sr["n_points"] != o["n_points"]:
            bad.append((i, "n_points", o["n_points"], int(sr["n_points"])))
        c = cands[sr["first_candidate"] : sr["first_candidate"] + sr["n_candidates"]]
        rl1 = o["l1"]
        same = len(c) == len(rl1) and all(
            np.array_equal(c[f], rl1[f]) for f in ("seqId", "rangeStartPos", "rangeEndPos", "intersectionSize"))
        if not same:
            bad.append((i, "l1", rl1.tolist(), c[["seqId", "rangeStartPos", "rangeEndPos", "intersectionSize"]].tolist()))
            o2 = R.map_fragment(d["rnames"][ridx[i]], seg, full_len=len(r), seq_counter=int(ridx[i]))
            print(f"DIAG seg {i}: reference minimumHits {o['minimumHits']} n_points {o['n_points']}; reference again l1 "
                  f"{o2['l1'].tolist()} minimumHits {o2['minimumHits']}; device minimum_hits {sr['minimum_hits']} best "
                  f"{sr['best_intersection']} n_points {sr['n_points']} sketch_size {sr['sketch_size']}")
            if diag is not None:
                diag(i, seg, len(r), int(ridx[i]), o)
            continue
        for ci in range(len(c)):
            dl = loci[c[ci]["first_locus"] : c[ci]["first_locus"] + c[ci]["n_loci"]]
            rl = o["l2"][o["l2_cand"] == ci]
            n_cmp += 1
            if len(dl) != len(rl) or not all(np.array_equal(dl[f], rl[f]) for f in rl.dtype.names):
                bad.append((i, f"l2 cand {ci}", rl.tolist(), dl.tolist()))
    for b in bad[:max_report]:
        print("MISMATCH", b)
    print(f"segments={len(ridx)} candidates_compared={n_cmp} mismatches={len(bad)}")
    golden_ref.check_stored("fragments", R.key, ref_digests)
    return bad


@pytest.fixture(scope="module")
def random_set(workdir):
    return datasets.make_random_set(workdir)


@pytest.fixture(scope="module")
def panel_set(workdir):
    return datasets.make_panel_set(workdir)


@pytest.mark.parametrize("mode", ["fast+general", "general-only"])
@pytest.mark.parametrize("k,s", [(19, 130), (16, 40), (21, 250), (32, 17)])
def test_sketch_matches_reference(random_set, k, s, mode, monkeypatch):
    """both sketch kernels: the one-pass fast kernel (its rejects go to the general kernel) and the general kernel alone"""
    from mashmap_b200 import capi

    if mode == "general-only":
        monkeypatch.setenv("MM_SKETCH_TABLE", "1")
    d = random_set
    ctx = capi.Context(kmer_size=k, seg_length=5000, sketch_size=s)
    bases, segs, ridx, start, length = build_segments(d, 5000, k)
    out, cnt = ctx.sketch_segments(bases, segs)
    want = reference_sketch_digests("sketch_random_set", f"k{k} s{s}", [d["reads"][ridx[i]][start[i] : start[i] + length[i]]
                                    for i in range(len(segs))], k, s, [int(x) for x in ridx])
    bad = 0
    for i in range(len(segs)):
        dev = out[i][: cnt[i]]
        ok = golden_ref.sketch_digest(dev) == want[i] and np.all(dev["seqId"] == ridx[i])
        if not ok:
            bad += 1
            if bad <= 5:
                print("sketch mismatch seg", i, "len", length[i], "dev n", len(dev))
    assert bad == 0
    ctx.close()


def degenerate_sequences():
    rng = np.random.default_rng(5)
    seqs = [np.full(5000, ord("N"), np.uint8), np.full(5000, ord("A"), np.uint8),
            np.tile(np.frombuffer(b"ACGTTGCAAG", np.uint8), 500), np.tile(synth.random_sequence(300, rng), 17)[:5000],
            synth.random_sequence(19, rng), synth.random_sequence(18, rng), synth.random_sequence(57, rng),
            synth.random_sequence(4999, rng), np.frombuffer(b"acgtnACGTRYKM" * 300, np.uint8)]
    mixed = synth.random_sequence(5000, rng)
    mixed[100:140] = ord("N"); mixed[4990:] = ord("N"); mixed[0] = ord("N")
    seqs.append(mixed)
    pal = synth.random_sequence(2500, rng)
    seqs.append(np.concatenate([pal, synth.revcomp(pal)]))  # every k-mer occurs on both strands -> vote sums of 0
    return seqs


def test_sketch_degenerate_inputs():
    """all-N, low-complexity (fewer than s distinct k-mers), tandem repeats, tiny and ragged segments"""
    from mashmap_b200 import capi

    k, s, L = 19, 100, 5000
    seqs = degenerate_sequences()
    ctx = capi.Context(kmer_size=k, seg_length=L, sketch_size=s)
    segs = np.zeros(len(seqs), dtype=capi.segment_dtype)
    off = 0
    for i, q in enumerate(seqs):
        segs[i]["offset"] = off; segs[i]["length"] = len(q); segs[i]["seq_counter"] = i; segs[i]["name_id"] = -1
        off += len(q)
    out, cnt = ctx.sketch_segments(np.concatenate(seqs), segs)
    want = reference_sketch_digests("sketch_degenerate", f"k{k} s{s}", seqs, k, s, list(range(len(seqs))))
    for i, q in enumerate(seqs):
        assert golden_ref.sketch_digest(out[i], cnt[i]) == want[i], i
    # homopolymers, tandem repeats, all-N, fewer than s distinct k-mers: the fast kernel must have handed them over
    dg = ctx.diag()
    print("rare paths taken:", dg)
    assert dg["sketch_general_segments"] >= 4
    ctx.close()


@pytest.fixture(params=["fast-paths", "general-kernels"])
def kernel_paths(request, monkeypatch):
    """the warp-per-segment L1 + stream L2 kernels (default), or the general CTA / warp-per-candidate kernels alone"""
    if request.param == "general-kernels":
        monkeypatch.setenv("MM_SKETCH_TABLE", "1")
        monkeypatch.setenv("MM_L1_CTA", "1")
        monkeypatch.setenv("MM_L2_GENERAL", "1")
    return request.param


def run_stage_parity(d, args, seg_length, expect_diag=(), expect_freq_seeds=False, check=None, **ctx_kw):
    """expect_diag: names of mm_ctx_diag counters that must be non-zero afterwards (the rare path really ran);
    expect_freq_seeds: the reference must have flagged frequent seeds and some query sketch must have lost hashes to them;
    check: called with the device's (segment results, candidates, loci)"""
    from mashmap_b200 import capi

    R = open_session(args, d)
    try:
        ctx = capi.Context(kmer_size=R.p.kmerSize, seg_length=R.p.segLength, sketch_size=R.p.sketchSize,
                           stage1_topani_filter=bool(R.p.stage1_topANI_filter), **ctx_kw)
        upload_reference_index(ctx, R)
        bases, segs, ridx, start, length = build_segments(d, R.p.segLength, R.p.kmerSize)
        seg_res, cands, loci = ctx.map_segments(bases, segs)
        # resident path must give the same answer
        ctx.batch_upload(bases, segs)
        ctx.map_resident()
        seg_res2, cands2, loci2 = ctx.batch_fetch()
        dev_sketch, dev_count = ctx.batch_fetch_sketch()
        # the first call is the one a fresh context's small buffers make regrow: its candidates and loci, fragment by
        # fragment, must be the resident call's, which is compared with the reference below
        first = [device_fragment_digest(i, seg_res, cands, loci, dev_sketch, dev_count) for i in range(len(segs))]
        assert first == [device_fragment_digest(i, seg_res2, cands2, loci2, dev_sketch, dev_count) for i in range(len(segs))], \
            "mm_map_segments and the resident path differ"
        print("stage ms", ctx.stage_ms(), "launches", ctx.kernel_launches)
        def diag(i, seg, full_len, counter, o):
            import oracle_py

            sr1 = seg_res[i]
            c1 = cands[sr1["first_candidate"] : sr1["first_candidate"] + sr1["n_candidates"]]
            print("   first (host-buffer) call gave", c1[["seqId", "rangeStartPos", "rangeEndPos", "intersectionSize"]].tolist())
            if oracle_py.available() and isinstance(R, refh.RefSession):
                O = oracle_py.Oracle(params=R.p)
                idx = R.index()
                keys, offs, pts, fr = R.lookup()
                O.set_index(idx, keys, offs, pts, fr, R.contig_len, R.contig_names)
                b = O.map_fragment(seg, seq_counter=counter, full_len=full_len)
                print("   oracle on the same index:", b["l1"].tolist(), "minimumHits", b["minimumHits"], "n_points", b["n_points"],
                      "points equal reference:", np.array_equal(o["points"], b["points"]))
                O.close()

        bad = compare_stages(ctx, R, d, ridx, start, length, seg_res2, cands2, loci2, dev_sketch, dev_count, diag=diag)
        if check is not None:
            check(seg_res2, cands2, loci2)
        dg = ctx.diag()
        print("rare paths taken:", dg)
        for name in expect_diag:
            assert dg[name] > 0, f"the test data no longer reaches the {name} path: {dg}"
        if expect_freq_seeds:
            fr = R.lookup()[3]
            removed = int((seg_res2["sketch_raw_count"] - seg_res2["sketch_size"]).sum())
            print(f"frequent seeds: threshold {R.freq_threshold()}, {int(np.asarray(fr).sum())} keys flagged, "
                  f"{removed} hashes removed from the query sketches on the device")
            assert np.asarray(fr).sum() > 0 and removed > 0
        ctx.close()
        return bad
    finally:
        R.close()


def test_stages_random_genome_noisy_reads(random_set, kernel_paths):
    d = random_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "4"], 5000)
    assert not bad


def test_stages_random_genome_dense(random_set, kernel_paths):
    d = random_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "95", "--dense", "-t", "4"], 5000)
    assert not bad


def test_stages_panel_selfmap(panel_set, kernel_paths):
    d = panel_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "4"], 5000)
    assert not bad


def test_stages_panel_no_hg_filter_small_sketch(panel_set, kernel_paths):
    d = panel_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "2000", "--pi", "90", "-J", "25", "--noHgFilter", "-t", "4"], 2000)
    assert not bad


def test_packed_input_equals_text_input(random_set):
    """mm_map_segments_packed (one nibble per base, the format a packing host uploads) == mm_map_segments (text, packed
    on the device by k_pack_bases): lower case, IUPAC codes, N runs and an all-N read are in the set"""
    from mashmap_b200 import capi

    d = random_set
    R = open_session(["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "4"], d)
    try:
        ctx = capi.Context(kmer_size=R.p.kmerSize, seg_length=R.p.segLength, sketch_size=R.p.sketchSize)
        upload_reference_index(ctx, R)
        bases, segs, ridx, start, length = build_segments(d, R.p.segLength, R.p.kmerSize)
        def canon(res):
            """per segment: (sketch size, points, minimum hits, candidates with their loci) -- the position of a segment's
            candidate slice in the batch-wide arrays depends on the order the CTAs reserved them in"""
            seg_res, cands, loci = res
            out = []
            for sr in seg_res:
                c = cands[sr["first_candidate"] : sr["first_candidate"] + sr["n_candidates"]]
                cl = [(tuple(int(x[f]) for f in ("seqId", "rangeStartPos", "rangeEndPos", "intersectionSize")),
                       loci[x["first_locus"] : x["first_locus"] + x["n_loci"]].tobytes()) for x in c]
                out.append((int(sr["sketch_max_hash"]), int(sr["sketch_raw_count"]), int(sr["sketch_size"]), int(sr["n_points"]),
                            int(sr["minimum_hits"]), int(sr["best_intersection"]), cl))
            return out

        a = canon(ctx.map_segments(bases, segs))
        assert ctx.pack_ms() > 0.0    # text input: packed on the device
        b = canon(ctx.map_segments_packed(capi.pack_bases(bases), len(bases), segs))
        assert a == b
        assert ctx.pack_ms() == 0.0  # the packed batch skipped the device packing kernel
        # odd segment offsets / an odd number of bases: shift everything by one base
        bases1 = np.concatenate([np.frombuffer(b"G", np.uint8), bases])
        segs1 = segs.copy()
        segs1["offset"] += 1
        c = canon(ctx.map_segments_packed(capi.pack_bases(bases1), len(bases1), segs1))
        assert a == c
        ctx.close()
    finally:
        R.close()


def every_k_subset(d):
    return dict(reads=d["reads"][:6] + d["reads"][-5:], rnames=d["rnames"][:6] + d["rnames"][-5:])


@pytest.mark.parametrize("k", list(range(8, 33)))
def test_sketch_every_kmer_size(random_set, k):
    """the reference accepts any -k (parseCmdArgs.hpp:435-443); every k-mer length from 8 to 32 is compiled in"""
    from mashmap_b200 import capi

    s = 60
    ctx = capi.Context(kmer_size=k, seg_length=3000, sketch_size=s)
    sub = every_k_subset(random_set)
    bases, segs, ridx, start, length = build_segments(sub, 3000, k)
    out, cnt = ctx.sketch_segments(bases, segs)
    want = reference_sketch_digests("sketch_every_k", f"k{k} s{s}", [sub["reads"][ridx[i]][start[i] : start[i] + length[i]]
                                    for i in range(len(segs))], k, s, [int(x) for x in ridx])
    for i in range(len(segs)):
        assert golden_ref.sketch_digest(out[i], cnt[i]) == want[i], (k, i)
    ctx.close()


def test_stages_frequent_seeds_removed_on_device(panel_set, kernel_paths):
    """--kmerThreshold high enough that the reference reports "ignore minmers occurring >= N": Sketch::isFreqSeed hashes are
    dropped from the query sketch on the device (table value bit 0; computeMap.hpp:834-839) and Q.sketchSize shrinks"""
    d = panel_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "--kmerThreshold", "5", "-t", "4"], 5000,
                           expect_freq_seeds=True)
    assert not bad


@pytest.fixture(scope="module")
def assembly_set(workdir):
    return datasets.make_assembly_set(workdir)


@pytest.fixture(scope="module")
def hifi_set(workdir):
    return datasets.make_hifi_set(workdir)


@pytest.fixture(scope="module")
def big_random_set(workdir):
    return datasets.make_big_random_set(workdir)


@pytest.fixture(scope="module")
def repeat_set(workdir):
    return datasets.make_repeat_set(workdir)


def test_stages_config5_shape_assembly_s10000(assembly_set, kernel_paths):
    """BASELINE config 5 shape: assembly vs assembly, -s 10000 --pi 90 -f one-to-one (10 kb fragments, automatic sketch)"""
    d = assembly_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "10000", "--pi", "90", "-f", "one-to-one", "-t", "4"], 10000)
    assert not bad


def test_stages_config4_shape_hifi_sketch20(hifi_set, kernel_paths):
    """BASELINE config 4 shape: 20 kb HiFi-like reads, --pi 95, sketch size 20 (what the reference picks for a 3 Gbp file)"""
    d = hifi_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "95", "-J", "20", "-f", "one-to-one", "-t", "4"], 5000)
    assert not bad


def test_stages_config3_shape_dense_pi95_32mbp(big_random_set):
    """BASELINE config 3 shape: --dense --pi 95 (s = 199) on a 32 Mbp reference"""
    d = big_random_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "95", "--dense", "-t", "8"], 5000)
    assert not bad


def test_stages_config2_shape_pi85_32mbp(big_random_set):
    d = big_random_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-J", "220", "-t", "8"], 5000)
    assert not bad


def test_stages_repeat_dense_l1_pool(repeat_set, monkeypatch):
    """fragments with 60-110 thousand interval points: more than the warp path (512), the CTA's shared memory (2048) and
    its global slice (65,536) hold -> bump-allocated pool; with a pool of 4,096 points the host has to grow it and re-run"""
    monkeypatch.setenv("MM_L1_POOL_ELEMS", "4096")
    d = repeat_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "4"], 5000,
                           expect_diag=("l1_cta_segments", "l1_pool_regrow"))
    assert not bad


def test_stages_repeat_dense_many_loci_per_candidate(repeat_set, kernel_paths):
    """without the hypergeometric filter one L1 candidate spans the whole tandem array and L2 returns six equally good loci
    (two fixed slots in the stream kernel -> general L2 kernel); the interspersed-repeat fragments scan a 2 Mbp range"""
    d = repeat_set
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "--noHgFilter", "-t", "4"], 5000,
                           expect_diag=("l2_general_cands",) if kernel_paths == "fast-paths" else ())
    assert not bad
