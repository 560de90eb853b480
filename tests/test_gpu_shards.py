"""--indexShards on the GPU: a reference index cut by contig into N device images gives the unsharded result.

- index: each shard's image is the unsharded image restricted to its contigs (minmers, interval points, keys, frequent
  flags), with global seqIds; the frequent hashes of the whole reference that a shard lacks are flagged keys with no points.
- stages: the per-segment records of all shards, merged in shard order, equal the unsharded context's field by field, on
  the fast kernels and on the general ones, with and without the HG filter, with fragments longer than a segment.
- CLI: the PAF of `--indexShards 2` and `3` is byte-identical to the unsharded run's for every command line of
  test_gpu_cli.py and the --noSplit ones of test_gpu_nosplit.py (which compare the unsharded PAF with the reference's),
  and on a reference whose frequent seeds a per-shard threshold would get wrong.
"""
import os
import subprocess

import numpy as np
import pytest

import datasets
import nosplit_data as ND
import shard_data as S
from conftest import have_gpu
from mashmap_b200 import capi, hostlib, synth

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_gpu(), reason="no GPU")]


# ---- index -------------------------------------------------------------------------------------------------------------

def shard_inputs(genome, first, i):
    seqs = genome[first[i] : first[i + 1]]
    return np.concatenate(seqs).astype(np.uint8), S.offsets(seqs)


def build_shards(genome, first, pct, params, keep_lookup=False, groups=None):
    """pass 1 on every shard, the host merge, pass 2: (contexts, threshold, frequent hashes)"""
    clen = np.array([len(c) for c in genome], dtype=np.int32)
    ctxs, ks, cs = [], [], []
    for i in range(len(first) - 1):
        ctx = capi.Context(**params)
        keys, counts, _ = ctx.index_key_counts(*shard_inputs(genome, first, i))
        ks.append(keys)
        cs.append(counts)
        ctxs.append(ctx)
    t, _, freq = hostlib.global_frequent_seeds(ks, cs, pct)
    for i, ctx in enumerate(ctxs):
        bases, offs = shard_inputs(genome, first, i)
        ctx.index_build_shard(bases, offs, first[i], clen, freq, contig_group=groups, keep_lookup=keep_lookup)
    return ctxs, t, freq


def key_points(keys, offs, pts):
    return {int(k): pts[int(offs[j]) : int(offs[j + 1])] for j, k in enumerate(keys)}


@pytest.mark.parametrize("n", [2, 3, 5])
def test_shard_images_are_the_unsharded_image_restricted(workdir, n):
    d = datasets.make_panel_set(workdir, tag="clip")
    genome, pct = d["genome"], 5.0
    params = dict(kmer_size=19, seg_length=5000, sketch_size=200)
    whole = capi.Context(**params)
    st = whole.index_build(np.concatenate(genome), S.offsets(genome), kmer_pct_threshold=pct, keep_lookup=True)
    mi, keys, offs, pts, fr = whole.index_download()
    whole.close()
    first = hostlib.plan_shards([len(c) for c in genome], np.zeros(len(genome), np.int32), False, n)
    ctxs, t, freq = build_shards(genome, first, pct, params, keep_lookup=True)
    assert t == st["freq_threshold"] and len(freq) == int(fr.sum()) > 0
    assert set(freq.tolist()) == set(keys[fr.astype(bool)].tolist())
    want = key_points(keys, offs, pts)
    freq_set = set(freq.tolist())
    n_absent = 0
    for i, ctx in enumerate(ctxs):
        lo, hi = first[i], first[i + 1]
        smi, skeys, soffs, spts, sfr = ctx.index_download()
        inside = (mi["seqId"] >= lo) & (mi["seqId"] < hi)
        assert np.array_equal(smi, mi[inside]), f"shard {i}: minmers"
        got = key_points(skeys, soffs, spts)
        assert len(got) == len(skeys)
        for j, k in enumerate(skeys.tolist()):
            p = want[k]
            exp = p[(p["seqId"] >= lo) & (p["seqId"] < hi)]
            assert np.array_equal(got[k], exp), f"shard {i}: points of {k:#x}"
            assert bool(sfr[j]) == (k in freq_set), f"shard {i}: flag of {k:#x}"
            if len(exp) == 0:  # a frequent hash of the reference that this shard lacks
                assert sfr[j] == 1
                n_absent += 1
        own = {k for k, p in want.items() if ((p["seqId"] >= lo) & (p["seqId"] < hi)).any()}
        assert own | freq_set == set(skeys.tolist()), f"shard {i}: keys"
        ctx.close()
    assert n_absent > 0


# ---- stages ------------------------------------------------------------------------------------------------------------

def merge(per_shard, n_segs):
    """the shards' records per segment in shard order, as skch::BatchMapper merges them"""
    seg_out = np.zeros(n_segs, dtype=capi.segres_dtype)
    cands, loci = [], []
    for s in range(n_segs):
        r = per_shard[0][0][s].copy()
        for f in ("sketch_max_hash", "sketch_raw_count", "sketch_size"):
            assert all(sr[s][f] == r[f] for sr, _, _ in per_shard), (s, f)
        r["first_candidate"], r["n_candidates"], r["n_points"], r["best_intersection"] = len(cands), 0, 0, 0
        mh = None
        for sr, c, l in per_shard:
            q = sr[s]
            r["n_points"] += q["n_points"]
            r["best_intersection"] = max(r["best_intersection"], q["best_intersection"])
            if mh is None and q["n_points"] > 0:
                mh = q["minimum_hits"]
            for cd in c[q["first_candidate"] : q["first_candidate"] + q["n_candidates"]]:
                cd = cd.copy()
                loci.extend(l[cd["first_locus"] : cd["first_locus"] + cd["n_loci"]])
                cd["first_locus"] = len(loci) - cd["n_loci"]
                cands.append(cd)
                r["n_candidates"] += 1
        r["minimum_hits"] = 0 if mh is None else mh
        seg_out[s] = r
    return seg_out, np.array(cands, dtype=capi.l1_dtype), np.array(loci, dtype=capi.l2_dtype)


def per_segment(seg_res, cands, loci):
    """each segment's result fields, its candidates and each candidate's loci (where the device put a segment's
    candidates in the array depends on the order its blocks ran)"""
    out = []
    for r in seg_res:
        fields = tuple(int(r[f]) for f in r.dtype.names if f not in ("first_candidate", "_pad"))
        cl = []
        for cd in cands[int(r["first_candidate"]) : int(r["first_candidate"]) + int(r["n_candidates"])]:
            ls = loci[int(cd["first_locus"]) : int(cd["first_locus"]) + int(cd["n_loci"])]
            cl.append((tuple(int(cd[f]) for f in cd.dtype.names if f not in ("first_locus", "_pad")),
                       [tuple(int(v) for v in x.tolist()) for x in ls]))
        out.append((fields, cl))
    return out


def segments(reads, seg, k, whole):
    lens = [len(r) for r in reads]
    offs = np.zeros(len(lens) + 1, dtype=np.int64)
    offs[1:] = np.cumsum(lens)
    if whole:  # every query one fragment: those longer than a segment take k_l1_long / k_l2_long
        ridx, start, length = np.arange(len(lens)), np.zeros(len(lens), np.int64), np.array(lens)
    else:
        ridx, start, length = synth.split_segments(lens, seg, k)
    sg = np.zeros(len(ridx), dtype=capi.segment_dtype)
    sg["offset"] = offs[ridx] + start
    sg["length"] = length
    sg["seq_counter"] = ridx
    sg["name_id"] = -1
    sg["ref_group"] = -1
    return np.concatenate(reads).astype(np.uint8), sg


@pytest.fixture(params=["fast-paths", "general-kernels"])
def kernel_paths(request, monkeypatch):
    if request.param == "general-kernels":
        monkeypatch.setenv("MM_SKETCH_TABLE", "1")
        monkeypatch.setenv("MM_L1_CTA", "1")
        monkeypatch.setenv("MM_L2_GENERAL", "1")
    return request.param


STAGE_CASES = [(w, hg, whole, n) for w, hg, whole in (("random", True, False), ("random", False, False), ("panel", True, True),
                                                 ("panel", False, True)) for n in (2, 3, 5)] + [("repeat", True, False, 2)]


@pytest.mark.parametrize("which,hg,whole,n", STAGE_CASES)
def test_merged_stages_equal_unsharded(workdir, kernel_paths, which, hg, whole, n):
    compare_sharded(workdir, which, hg, whole, n)


def compare_sharded(workdir, which, hg, whole, n):
    """the merged stages of n shards against the unsharded context's; returns each shard context's diag counters"""
    make = {"random": lambda: datasets.make_big_random_set(workdir, tag="shbig"),
            "repeat": lambda: datasets.make_repeat_set(workdir, tag="clir"),
            "panel": lambda: datasets.make_panel_set(workdir, tag="clip")}[which]
    d = make()
    genome = d["genome"]
    k, seg, s, pct, pi = 19, 5000, 200, 0.5, 0.85
    params = dict(kmer_size=k, seg_length=seg, sketch_size=s, stage1_topani_filter=hg)
    tables = (hostlib.sketch_cutoffs(s, k, enabled=hg), hostlib.min_hits_table(s, k, pi))
    bases, sg = segments(d["reads"], seg, k, whole)

    ref = capi.Context(**params)
    ref.index_build(np.concatenate(genome), S.offsets(genome), kmer_pct_threshold=pct)
    ref.tables_upload(*tables)
    want = ref.map_segments(bases, sg)
    ref.close()

    first = hostlib.plan_shards([len(c) for c in genome], np.zeros(len(genome), np.int32), False, n)
    ctxs, _, _ = build_shards(genome, first, pct, params)
    for c in ctxs:
        c.tables_upload(*tables)
        c.batch_upload(bases, sg)
    bests = [c.map_resident_l1_best() for c in ctxs]
    best = np.max(bests, axis=0)
    for i, c in enumerate(ctxs):
        after = np.zeros(len(sg), dtype=np.uint8)
        for later in bests[i + 1 :]:
            after |= (later > 0).astype(np.uint8)
        c.map_resident_with_best(best, after)
    got = merge([c.batch_fetch() for c in ctxs], len(sg))
    diags = [c.diag() for c in ctxs]
    if whole:
        assert any(dg["long_fragments"] > 0 for dg in diags)
    for c in ctxs:
        c.close()
    w, g = per_segment(*want), per_segment(*got)
    bad = [i for i in range(len(sg)) if w[i] != g[i]]
    assert not bad, (len(bad), w[bad[0]], g[bad[0]]) if bad else None
    assert want[0]["n_candidates"].sum() > 0
    return diags


def test_given_best_needs_its_first_phase():
    ctx = capi.Context(kmer_size=19, seg_length=1000, sketch_size=40, skip_prefix=True)
    genome = synth.random_genome(2, 30_000, seed=5)
    ctx.index_build(np.concatenate(genome), S.offsets(genome))
    ctx.tables_upload(hostlib.sketch_cutoffs(40, 19), hostlib.min_hits_table(40, 19, 0.85))
    bases, sg = segments([g[:3000] for g in genome], 1000, 19, False)
    ctx.batch_upload(bases, sg)
    with pytest.raises(capi.MashmapError, match="skip_prefix"):
        ctx.map_resident_l1_best()
    with pytest.raises(capi.MashmapError, match="has not run"):
        ctx.map_resident_with_best(np.zeros(len(sg), np.int32), np.zeros(len(sg), np.uint8))
    ctx.close()


# ---- CLI ---------------------------------------------------------------------------------------------------------------

def run(cmd):
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 0, (cmd, p.stderr[-3000:])
    return p.stderr


def index_lines(log):
    return [x for x in log.splitlines() if "computeFreqHist" in x or "unique minmers" in x or "windows picked" in x]


CLI = [  # test_gpu_cli.py's CONFIGS, then test_gpu_nosplit.py's command lines
    ("random", ["-s", "5000", "--pi", "85"]),
    ("random", ["-s", "5000", "--pi", "95", "--dense"]),
    ("random", ["-s", "5000", "--pi", "85", "-f", "none", "--noMerge"]),
    ("panel", ["-s", "5000", "--pi", "85"]),
    ("panel", ["-s", "5000", "--pi", "95", "-n", "1", "-Y", "#"]),
    ("panel", ["-s", "3000", "--pi", "90", "-f", "one-to-one", "-X"]),
    ("panel", ["-s", "5000", "--pi", "90", "--lowerTriangular", "-n", "2"]),
    ("panel", ["-s", "2000", "--pi", "90", "-J", "25", "--noHgFilter", "-k", "16"]),
    ("panel", ["-s", "5000", "--pi", "85", "--kmerThreshold", "5"]),
    ("panel", ["-s", "3000", "--pi", "90", "-k", "14", "-J", "40"]),
    ("assembly", ["-s", "10000", "--pi", "90", "-f", "one-to-one"]),
    ("hifi", ["-s", "5000", "--pi", "95", "-J", "20", "-f", "one-to-one"]),
    ("repeat", ["-s", "5000", "--pi", "85"]),
    ("repeat", ["-s", "5000", "--pi", "85", "--noHgFilter", "-n", "4"]),
] + [(w, ["--noSplit"] + a) for w, a in ND.CLI_RUNS]
MAKERS = {"random": ("cli", datasets.make_random_set), "panel": ("clip", datasets.make_panel_set),
          "assembly": ("clia", datasets.make_assembly_set), "hifi": ("clih", datasets.make_hifi_set),
          "repeat": ("clir", datasets.make_repeat_set)}


@pytest.mark.parametrize("which,args", CLI)
def test_cli_paf_is_identical_with_index_shards(workdir, which, args):
    d = MAKERS[which][1](workdir, tag=MAKERS[which][0])
    tag = "_".join(a.strip("-#") for a in args)
    base = os.path.join(workdir, f"sh1_{which}_{tag}.paf")
    log1 = run([hostlib.CLI_PATH, "-r", d["ref"], "-q", d["qry"], "-t", "8", "-o", base] + args)
    want = open(base, "rb").read()
    assert len(want) > 0
    n_ok = 0
    for n in (2, 3):
        if n > len(d["genome"]):
            continue
        out = os.path.join(workdir, f"sh{n}_{which}_{tag}.paf")
        log = run([hostlib.CLI_PATH, "-r", d["ref"], "-q", d["qry"], "-t", "8", "--indexShards", str(n), "-o", out] + args)
        assert open(out, "rb").read() == want, f"--indexShards {n}"
        assert index_lines(log) == index_lines(log1)
        n_ok += 1
    assert n_ok > 0


def test_cli_global_frequent_seeds(workdir):
    """a repeat element below the frequency threshold in every shard and above it over the whole reference"""
    d = S.write_set(workdir)
    first = hostlib.plan_shards([len(c) for c in d["genome"]], np.zeros(S.N_CONTIGS, np.int32), False, 2)
    pct = S.pick_pct(d["genome"], list(first))
    args = ["-s", str(S.SEG), "-J", str(S.SKETCH), "--pi", "85", "--kmerThreshold", repr(pct), "-t", "4"]
    base = os.path.join(workdir, "gf1.paf")
    log1 = run([hostlib.CLI_PATH, "-r", d["ref"], "-q", d["qry"], "-o", base] + args)
    want = open(base, "rb").read()
    assert len(want) > 0 and "ignore minmers occurring" in log1
    for n in (2, 3, 4):
        out = os.path.join(workdir, f"gf{n}.paf")
        log = run([hostlib.CLI_PATH, "-r", d["ref"], "-q", d["qry"], "--indexShards", str(n), "-o", out] + args)
        assert index_lines(log) == index_lines(log1)
        assert open(out, "rb").read() == want, f"--indexShards {n}"


@pytest.mark.skipif(not have_gpu() or __import__("torch").cuda.device_count() < 2, reason="one GPU")
def test_cli_two_devices(workdir):
    d = datasets.make_panel_set(workdir, tag="clip")
    args = ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "8"]
    a, b = os.path.join(workdir, "dev1.paf"), os.path.join(workdir, "dev2.paf")
    run([hostlib.CLI_PATH] + args + ["-o", a])
    run([hostlib.CLI_PATH] + args + ["--devices", "0,1", "--indexShards", "2", "-o", b])
    assert open(a, "rb").read() == open(b, "rb").read()
