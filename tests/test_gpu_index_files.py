"""--saveIndex and --loadIndex on the device. The builder keeps the records before the frequent-seed drop and the lookup
(MM_KEEP_UNFILTERED | MM_KEEP_LOOKUP) for the files, and a loaded minmer list is indexed by mm_index_build_minmers. The
files and the PAF must equal those of the host path (--hostIndex --saveIndex / --loadIndex), and a file whose records do
not fit the reference is refused before the device indexes anything by them."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import datasets
import refh
from conftest import have_gpu
from mashmap_b200 import capi, hostlib, synth

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_gpu(), reason="no GPU")]


def run(cmd, status=0):
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == status, (cmd, p.returncode, p.stderr[-2000:])
    return p.stderr


def cli(args, out, *extra, status=0):
    return run([hostlib.CLI_PATH] + args + list(extra) + ["-o", out], status)


def data(path):
    with open(path, "rb") as f:
        return f.read()


def read_index(path):
    raw = data(path)
    n = int(np.frombuffer(raw[:8], dtype=np.uint64)[0])
    return np.frombuffer(raw[8:8 + 24 * n], dtype=capi.minmer_dtype).copy()


def map_bytes(keys, offs, pts):
    """PREFIX.map as savePosListBinary writes it (keys ascending)"""
    out = [np.array([len(keys)], dtype=np.uint64).tobytes()]
    for i, k in enumerate(keys):
        a, b = int(offs[i]), int(offs[i + 1])
        out.append(np.array([k, b - a], dtype=np.uint64).tobytes())
        out.append(np.ascontiguousarray(pts[a:b]).tobytes())
    return b"".join(out)


def short_contig_set(workdir):
    """a random genome with contigs shorter than k (no records) and shorter than a window between the long ones"""
    ref, qry = os.path.join(workdir, "xs_ref.fa"), os.path.join(workdir, "xs_reads.fa")
    g = synth.random_genome(3, 200_000, seed=71)
    contigs = [g[0], g[1][:12], g[1][:150], g[2], g[1][12:19]]
    names = [f"c{i}" for i in range(len(contigs))]
    reads, _ = synth.simulate_reads([g[0], g[2]], 20, 8000, 0.02, 0.14, seed=72)
    synth.write_fasta(ref, names, contigs)
    synth.write_fasta(qry, [f"r{i}" for i in range(len(reads))], reads)
    return dict(ref=ref, qry=qry, genome=contigs)


SETS = {
    "random": (lambda w: datasets.make_random_set(w, tag="xr"), ["-s", "5000", "--pi", "85"]),
    "panel": (lambda w: datasets.make_panel_set(w, tag="xp"), ["-s", "5000", "--pi", "85", "--kmerThreshold", "5"]),
    "dense": (lambda w: datasets.make_random_set(w, tag="xd"), ["-s", "5000", "--pi", "95", "--dense"]),
    "k16": (lambda w: datasets.make_panel_set(w, tag="xk"), ["-s", "2000", "--pi", "90", "-k", "16"]),
    "short": (short_contig_set, ["-s", "1000", "--pi", "85"]),
}
_made = {}


def dataset(workdir, name):
    if name not in _made:
        make, opts = SETS[name]
        d = make(workdir)
        _made[name] = (d, ["-r", d["ref"], "-q", d["qry"], "-t", "4"] + opts)
    return _made[name]


@pytest.mark.parametrize("name", list(SETS))
def test_device_save_equals_host_save(workdir, name):
    d, args = dataset(workdir, name)
    base = os.path.join(workdir, f"sv_{name}")
    for ext in ("", ".tsv"):
        p, q = base + "_dev" + ext, base + "_host" + ext
        log = cli(args, p + ".paf", "--saveIndex", p)
        assert "index saved to" in log
        cli(args, q + ".paf", "--saveIndex", q, "--hostIndex")
        files = [(p, q)] if ext else [(p + ".index", q + ".index")]
        files.append((p + ".map", q + ".map"))
        for a, b in files:
            assert data(a) == data(b), (a, b)
        assert data(p + ".paf") == data(q + ".paf") and os.path.getsize(p + ".paf") > 0
        if name == "short":
            assert int(np.frombuffer(data(p + ".map")[:8], dtype=np.uint64)[0]) > 0


@pytest.mark.parametrize("w,s,k", [(1000, 20, 19), (500, 10, 16), (2000, 64, 21)])
def test_device_save_of_degenerate_contigs(workdir, monkeypatch, w, s, k):
    """On tandem repeats, N runs, low complexity and contigs shorter than k the saved records are the host window machine's
    under the device's tie rule (emission order) and the saved lookup is Sketch::index over them."""
    import test_host_cpu as t

    cases = t._cases_for_index()
    genome = [v if isinstance(v, np.ndarray) else np.frombuffer(bytes(v), dtype=np.uint8).copy() for v in cases.values()]
    ref = os.path.join(workdir, f"dg_{w}_{k}.fa")
    synth.write_fasta(ref, [f"g{i}" for i in range(len(genome))], genome)
    monkeypatch.setenv("MM_INDEX_CHUNK", str(max(1024, w // 2 * 3)))
    prefix = os.path.join(workdir, f"dg_{w}_{k}")
    cli(["-r", ref, "-q", ref, "-s", str(w), "-J", str(s), "-k", str(k), "--pi", "85", "-t", "4"], prefix + ".paf", "--saveIndex", prefix)
    want = np.concatenate([hostlib.add_minmers(g, k, w, s, seq_id=i, stable_ties=True) for i, g in enumerate(genome)])
    assert data(prefix + ".index") == np.array([len(want)], dtype=np.uint64).tobytes() + want.tobytes()
    hi = hostlib.HostIndex.from_minmers(want, len(genome))
    _, keys, offs, pts, _ = hi.arrays()
    hi.close()
    assert data(prefix + ".map") == map_bytes(keys, offs, pts)


def saved_records(workdir):
    d, args = dataset(workdir, "panel")
    p = os.path.join(workdir, "sv_panel_dev")
    if not os.path.exists(p + ".index"):
        cli(args, p + ".paf", "--saveIndex", p)
    return d, read_index(p + ".index")


def test_abi_load_from_host_and_device_memory(workdir):
    import torch

    d, mi = saved_records(workdir)
    clen = [len(c) for c in d["genome"]]
    hi = hostlib.HostIndex.from_minmers(mi, len(clen), 5.0)
    want = hi.arrays()
    threshold = hi.freq_threshold
    hi.close()
    assert threshold != 2**31 - 1 and len(want[0]) < len(mi)
    ctx = capi.Context(kmer_size=19, seg_length=5000, sketch_size=200)
    on_dev = torch.from_numpy(mi.view(np.uint8)).cuda()
    for ptr in (None, on_dev.data_ptr()):
        st = ctx.index_build_minmers(mi, clen, kmer_pct_threshold=5.0, keep_lookup=True, device_ptr=ptr)
        assert st["n_minmers_before_filter"] == len(mi) and st["n_chunks"] == 0 and st["freq_threshold"] == threshold
        got = ctx.index_download()
        for x, y in zip(got, want):
            for f in (x.dtype.names or [None]):
                if f is None:
                    assert np.array_equal(x, y)
                elif not f.startswith("_"):
                    assert np.array_equal(x[f], y[f]), f
    # what it keeps with MM_KEEP_UNFILTERED is its input, _pad zeroed
    junk = mi.copy()
    junk["_pad"] = 0x5a5a
    ctx.index_build_minmers(junk, clen, kmer_pct_threshold=5.0, keep_unfiltered=True)
    back = ctx.index_download_unfiltered()
    assert back.tobytes() == mi.tobytes() and np.all(back["_pad"] == 0)
    with pytest.raises(capi.MashmapError) as e:
        ctx.index_download_unfiltered()
    assert e.value.code == capi.MM_ESTATE
    ctx.close()


def test_cli_load_equals_host_load(workdir):
    d, args = dataset(workdir, "random")
    prefixes = []
    for ext in ("", ".tsv"):
        p = os.path.join(workdir, "ld_ours" + ext)
        cli(args, p + ".paf", "--saveIndex", p)
        prefixes.append(p)
        if os.path.exists(refh.REF_BIN):
            r = os.path.join(workdir, "ld_ref" + ext)
            run([refh.REF_BIN] + args + ["--saveIndex", r, "-o", r + ".paf"])
            prefixes.append(r)
    plain = os.path.join(workdir, "ld_plain.paf")
    cli(args, plain)
    assert data(plain) == data(os.path.join(workdir, "ld_ours.paf"))
    modes = [[], ["-f", "map"], ["-f", "one-to-one"], ["--noSplit"], ["--align"]]
    import torch

    if torch.cuda.device_count() >= 2:
        modes.append(["--devices", "0,1"])
    for p in prefixes:
        for m in (modes if not p.endswith(".tsv") else [[], ["--noSplit"]]):
            tag = os.path.basename(p) + "_" + "_".join(x.strip("-") for x in m)
            a, b = os.path.join(workdir, tag + "_dev.paf"), os.path.join(workdir, tag + "_host.paf")
            log = cli(args + m, a, "--loadIndex", p)
            assert "index built on the device from the" in log, log[-500:]
            cli(args + m, b, "--loadIndex", p, "--hostIndex")
            assert data(a) == data(b) and os.path.getsize(a) > 0, (p, m)
            if not m and p.endswith("ld_ours"):  # device save, then device load: the PAF of a plain run
                assert data(a) == data(plain)


@pytest.mark.parametrize("src_ext,dst_ext", [("", ""), ("", ".tsv"), (".tsv", "")])
def test_load_then_save_equals_host(workdir, src_ext, dst_ext):
    """--loadIndex P --saveIndex Q writes the loaded records and their lookup again, as the reference does after a load
    (winSketch.hpp:122-134): Q equals what --hostIndex --loadIndex P --saveIndex Q writes. That is how an index is turned
    from binary into TSV and back. From a file saved by the reference, whose records' _pad bytes are not initialised,
    the device writes them as zero and the host copies them: only they may differ."""
    d, args = dataset(workdir, "panel")
    sources = [("ours", os.path.join(workdir, "ls_ours" + src_ext))]
    cli(args, sources[0][1] + ".paf", "--saveIndex", sources[0][1])
    if os.path.exists(refh.REF_BIN):
        r = os.path.join(workdir, "ls_ref" + src_ext)
        run([refh.REF_BIN] + args + ["--saveIndex", r, "-o", r + ".paf"])
        sources.append(("ref", r))
    for who, p in sources:
        q, h = (os.path.join(workdir, f"ls_{who}{src_ext or '_bin'}_to{dst_ext or '_bin'}_{x}") + dst_ext for x in ("dev", "host"))
        log = cli(args, q + ".paf", "--loadIndex", p, "--saveIndex", q)
        assert "index built on the device from the" in log and "index saved to" in log, log[-800:]
        cli(args, h + ".paf", "--loadIndex", p, "--saveIndex", h, "--hostIndex")
        assert data(q + ".paf") == data(h + ".paf") and os.path.getsize(q + ".paf") > 0
        assert data(q + ".map") == data(h + ".map")
        if dst_ext:
            assert data(q) == data(h)
        elif who == "ours" or src_ext:
            assert data(q + ".index") == data(h + ".index")
        else:
            a, b = read_index(q + ".index"), read_index(h + ".index")
            assert len(a) == len(b) > 0 and np.all(a["_pad"] == 0)
            for f in ("hash", "wpos", "wpos_end", "seqId", "strand"):
                assert np.array_equal(a[f], b[f]), f


def test_an_upload_drops_what_a_build_kept(workdir):
    """what MM_KEEP_LOOKUP / MM_KEEP_UNFILTERED kept belongs to the index it was kept with: an mm_index_upload that
    replaces that index releases it"""
    d, mi = saved_records(workdir)
    clen = [len(c) for c in d["genome"]]
    ctx = capi.Context(kmer_size=19, seg_length=5000, sketch_size=200)
    ctx.index_build_minmers(mi, clen, keep_lookup=True, keep_unfiltered=True)
    arrays = ctx.index_download()
    ctx.index_upload(*arrays, clen)
    for call in (ctx.index_download_unfiltered, ctx.index_download):
        with pytest.raises(capi.MashmapError) as e:
            call()
        assert e.value.code == capi.MM_ESTATE
    ctx.close()


def test_bad_index_files_are_refused(workdir):
    d, args = dataset(workdir, "random")
    good = os.path.join(workdir, "bad_src")
    cli(args, good + ".paf", "--saveIndex", good)
    mi = read_index(good + ".index")
    assert len(mi) > 100 and mi["seqId"].max() == 2
    raw = data(good + ".index")

    def expect_refused(tag, blob, *words):
        p = os.path.join(workdir, "bad_" + tag)
        with open(p + ".index", "wb") as f:
            f.write(blob)
        shutil.copy(good + ".map", p + ".map")
        err = cli(args, p + ".paf", "--loadIndex", p, status=1)
        assert p + ".index" in err, err[-800:]
        for w in words:
            assert w in err, (w, err[-800:])

    expect_refused("truncated", raw[:-5], str(len(raw) - 5) + " bytes")
    huge = np.array([len(mi) * 1000], dtype=np.uint64).tobytes() + raw[8:]
    expect_refused("count", huge, str(len(raw)) + " bytes", str(len(mi) * 1000))
    expect_refused("short_header", raw[:5], "5 bytes")
    # saved from a longer reference: this one lacks the last contig
    short_ref = os.path.join(workdir, "bad_short_ref.fa")
    synth.write_fasta(short_ref, d["names"][:2], d["genome"][:2])
    first = int(np.argmax(mi["seqId"] == 2))
    p = os.path.join(workdir, "bad_longer")
    shutil.copy(good + ".index", p + ".index")
    shutil.copy(good + ".map", p + ".map")
    err = cli(["-r", short_ref] + args[2:], p + ".paf", "--loadIndex", p, status=1)
    assert p + ".index" in err and f"record {first}:" in err and "seqId 2" in err, err[-800:]
    i = int(np.nonzero((mi["seqId"][:-1] == mi["seqId"][1:]) & (mi["wpos"][:-1] < mi["wpos"][1:]))[0][10])
    unordered = mi.copy()
    unordered[[i, i + 1]] = unordered[[i + 1, i]]
    expect_refused("order", np.array([len(mi)], dtype=np.uint64).tobytes() + unordered.tobytes(), f"record {i + 1} ", "order")
    negative = mi.copy()
    negative["wpos"][77] = -3
    expect_refused("negative", np.array([len(mi)], dtype=np.uint64).tobytes() + negative.tobytes(), "record 77:", "negative")

    # through the ABI: MM_EINVAL, and the context then has no index (the good one it had is gone too)
    clen = [len(c) for c in d["genome"]]
    ctx = capi.Context(kmer_size=19, seg_length=5000, sketch_size=200)
    reads = d["reads"][0][:5000]
    segs = np.zeros(1, dtype=capi.segment_dtype)
    segs["length"] = len(reads)
    segs["name_id"] = -1
    segs["ref_group"] = -1
    for bad, n_contigs in ((unordered, 3), (negative, 3), (mi, 2)):
        ctx.index_build_minmers(mi, clen)
        ctx.tables_upload(hostlib.sketch_cutoffs(200, 19), hostlib.min_hits_table(200, 19, 0.85))
        ctx.map_segments(reads, segs)
        with pytest.raises(capi.MashmapError) as e:
            ctx.index_build_minmers(bad, clen[:n_contigs])
        assert e.value.code == capi.MM_EINVAL and "record" in str(e.value)
        with pytest.raises(capi.MashmapError) as e:
            ctx.map_segments(reads, segs)
        assert e.value.code == capi.MM_ESTATE
    ctx.close()
