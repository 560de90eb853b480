"""mashmap-b200 --align on the device: the NW mode of the C ABI per pair against edlib (oracle/_ref/libedlib_nw_ref.so,
or the full-matrix restatement oracle/libalign_nw_oracle.so where it is not built), mixed HW / NW batches, and the CLI on
synthetic cases: the PAF without the tags is the PAF of the same run without --align, every CIGAR consumes exactly the
mapping's region, and NM / cg equal edlib NW of the regions cut from the FASTA files here."""
import os
import re
import subprocess

import numpy as np
import pytest

import align_data as AD
import align_nw_data as AN
import datasets
from conftest import have_gpu
from mashmap_b200 import capi, synth

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_gpu(), reason="no GPU")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAP_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200")


def _jobs(pairs, modes):
    qb = np.concatenate([p[0] for p in pairs])
    tb = np.concatenate([p[1] for p in pairs])
    jobs = np.zeros(len(pairs), dtype=capi.align_job_dtype)
    jobs["q_len"] = [len(p[0]) for p in pairs]
    jobs["t_len"] = [len(p[1]) for p in pairs]
    jobs["q_offset"][1:] = np.cumsum(jobs["q_len"].astype(np.int64))[:-1]
    jobs["t_offset"][1:] = np.cumsum(jobs["t_len"].astype(np.int64))[:-1]
    jobs["k"] = [p[2] for p in pairs]
    jobs["mode"] = modes
    return qb, tb, jobs


def _result(res, ops, i):
    r = res[i]
    o = int(r["ops_offset"])
    return int(r["ed"]), int(r["start"]), int(r["end"]), ops[o : o + int(r["alignment_length"])]


def test_abi_nw_matches_edlib_on_random_pairs():
    """>= 50,000 pairs of the CPU tests' generators through mm_align_batch with MM_ALIGN_NW, in a few batches"""
    rng = np.random.default_rng(4242)
    check = AN.nw_check()
    ctx = capi.AlignContext(0)
    total = 0
    for batch in range(5):
        pairs = []
        for i in range(10_400):
            if i % 200 == 0:
                q, t = AD.threshold_pair(rng)
            elif i % 7 == 0:
                q, t = AN.long_indel_pair(rng)
            else:
                q, t = AD.random_pair(rng)
            r = rng.random()
            k = -1 if r < 0.4 else (max(len(q), len(t)) if r < 0.55 else int(rng.integers(0, max(1, len(q) // 2))))
            pairs.append((q, t, k))
        qb, tb, jobs = _jobs(pairs, capi.MM_ALIGN_NW)
        res, ops = ctx.align(qb, tb, jobs)
        for i, (q, t, k) in enumerate(pairs):
            want = check(q, t, k)
            got = _result(res, ops, i)
            assert got[:3] == tuple(want[:3]), (batch, i, len(q), len(t), k)
            assert np.array_equal(got[3], want[3]), (batch, i, len(q), len(t), k)
        total += len(pairs)
    assert total >= 50_000
    ctx.close()


def test_mixed_batches_leave_hw_results_unchanged():
    """HW jobs give the same results alone and interleaved with NW jobs on the same pairs; the NW jobs of the mixed batch
    give what they give alone"""
    rng = np.random.default_rng(77)
    pairs = []
    for i in range(3000):
        q, t = AD.threshold_pair(rng) if i % 100 == 0 else AD.random_pair(rng)
        pairs.append((q, t, -1 if i % 3 else len(q)))
    ctx = capi.AlignContext(0)
    modes = np.array([capi.MM_ALIGN_NW if i % 2 else capi.MM_ALIGN_HW for i in range(len(pairs))], dtype=np.int32)
    hw_idx = [i for i in range(len(pairs)) if modes[i] == capi.MM_ALIGN_HW]
    nw_idx = [i for i in range(len(pairs)) if modes[i] == capi.MM_ALIGN_NW]
    res_m, ops_m = ctx.align(*_jobs(pairs, modes))
    res_h, ops_h = ctx.align(*_jobs([pairs[i] for i in hw_idx], capi.MM_ALIGN_HW))
    res_n, ops_n = ctx.align(*_jobs([pairs[i] for i in nw_idx], capi.MM_ALIGN_NW))
    for j, i in enumerate(hw_idx):
        a, b = _result(res_m, ops_m, i), _result(res_h, ops_h, j)
        assert a[:3] == b[:3] and np.array_equal(a[3], b[3]), i
    for j, i in enumerate(nw_idx):
        a, b = _result(res_m, ops_m, i), _result(res_n, ops_n, j)
        assert a[:3] == b[:3] and np.array_equal(a[3], b[3]), i
        assert a[1:3] == (0, len(pairs[i][1]) - 1) or a[0] < 0
    ctx.close()


def test_abi_rejects_an_unknown_mode():
    ctx = capi.AlignContext(0)
    q = np.frombuffer(b"ACGTACGTAC", dtype=np.uint8)
    for mode in (2, -1):
        jobs = np.zeros(1, dtype=capi.align_job_dtype)
        jobs["q_len"], jobs["t_len"], jobs["k"], jobs["mode"] = 10, 10, -1, mode
        with pytest.raises(capi.MashmapError) as e:
            ctx.align(q, q, jobs)
        assert e.value.code == capi.MM_EINVAL and "mode" in str(e.value)
    ctx.close()


# ---- the CLI ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("map_align"))
    rnd = datasets.make_random_set(d, tag="ma", n_contigs=3, contig_len=300_000, n_reads=40, read_len=10_000, seed=71)
    # assembly-like: eight 25 kb contigs, the query a 3 % diverged copy with an inversion and a run of N
    rng = np.random.default_rng(72)
    genome = synth.random_genome(8, 25_000, seed=73)
    other = [synth.mutate(c, 0.03, rng, ratio=(30, 2, 1)) for c in genome]
    other[2] = np.concatenate([other[2][:8000], synth.revcomp(other[2][8000:16000]), other[2][16000:]])
    other[5] = other[5].copy()
    other[5][10_000:10_300] = ord("N")
    synth.write_fasta(os.path.join(d, "asm_a.fa"), [f"a{i}" for i in range(8)], genome)
    synth.write_fasta(os.path.join(d, "asm_b.fa"), [f"b{i}" for i in range(8)], other)
    return dict(dir=d, ref=rnd["ref"], qry=rnd["qry"], asm_ref=os.path.join(d, "asm_a.fa"),
                asm_qry=os.path.join(d, "asm_b.fa"))


CASES = {  # name -> (dataset, options)
    "ont_pi85": ("rnd", ["--pi", "85"]),
    "ont_f_none": ("rnd", ["--pi", "85", "-f", "none"]),
    "ont_nosplit": ("rnd", ["--pi", "85", "--noSplit"]),
    "asm_one_to_one": ("asm", ["--pi", "90", "-s", "2000", "-f", "one-to-one"]),
}


def _map(data, name, extra=(), tag=""):
    which, opts = CASES[name]
    ref, qry = (data["ref"], data["qry"]) if which == "rnd" else (data["asm_ref"], data["asm_qry"])
    out = os.path.join(data["dir"], f"{name}{tag}.paf")
    p = subprocess.run([MAP_BIN, "-r", ref, "-q", qry, "-o", out] + opts + list(extra), capture_output=True, text=True,
                       cwd=data["dir"])
    assert p.returncode == 0, p.stderr[-3000:]
    return open(out).read(), p.stderr


_aligned = {}


def _aligned_run(data, name):
    if name not in _aligned:
        _aligned[name] = _map(data, name, ["--align"], ".align")
    return _aligned[name]


@pytest.mark.parametrize("name", sorted(CASES))
def test_cli_tags_are_edlib_nw_of_each_region(data, name):
    plain, _ = _map(data, name)
    text, err = _aligned_run(data, name)
    assert plain.count("\n") > 5
    assert AN.strip_tags(text) == plain
    which, _ = CASES[name]
    fa = (data["qry"], data["ref"]) if which == "rnd" else (data["asm_qry"], data["asm_ref"])
    tagged, untagged = AN.check_tags(text, AN.read_fasta(fa[0]), AN.read_fasta(fa[1]))
    assert tagged == plain.count("\n") and untagged == 0
    assert re.search(rf"\] {tagged} mappings aligned", err), err[-2000:]
    assert "; 0 mappings with a region longer than --alignMaxLen 100000 " in err  # the default
    strands = {ln.split("\t")[4] for ln in text.splitlines()}
    assert strands == {"+", "-"}  # reads on both strands (the inversion for the assembly)
    if which == "rnd":  # read41 is a copy of a reference stretch with N runs
        assert any(ln.startswith("read41\t") for ln in text.splitlines())


@pytest.mark.parametrize("name", ["ont_pi85", "asm_one_to_one"])
def test_cli_output_does_not_depend_on_batches_or_threads(data, name):
    want, _ = _aligned_run(data, name)
    for extra in (["--batchBases", "30000", "--subBatchBases", "12000", "-t", "1"], ["-t", "8"]):
        got, _ = _map(data, name, ["--align"] + extra, ".b")
        assert got == want, extra


def _gpu_count():
    import torch

    return torch.cuda.device_count() if have_gpu() else 0


@pytest.mark.skipif(_gpu_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("name", ["ont_pi85", "asm_one_to_one"])
def test_cli_output_does_not_depend_on_devices(data, name):
    want, _ = _aligned_run(data, name)
    got, _ = _map(data, name, ["--align", "--devices", "0,1", "--subBatchBases", "30000"], ".dev")
    assert got == want


@pytest.mark.parametrize("name", ["ont_pi85", "asm_one_to_one"])
def test_cli_host_and_loaded_index_give_the_same_output(data, name):
    want, _ = _aligned_run(data, name)
    got, _ = _map(data, name, ["--align", "--hostIndex"], ".host")
    assert got == want
    idx = os.path.join(data["dir"], f"{name}.idx")
    saved, _ = _map(data, name, ["--align", "--saveIndex", idx], ".save")
    assert saved == want
    got, _ = _map(data, name, ["--align", "--loadIndex", idx], ".load")
    assert got == want


def test_cli_align_max_len_drops_the_tags_of_longer_mappings_only(data):
    want, _ = _aligned_run(data, "ont_pi85")
    lens = [max(int(f[3]) - int(f[2]), int(f[8]) - int(f[7])) for f in (ln.split("\t") for ln in want.splitlines())]
    limit = sorted(lens)[len(lens) // 2]
    got, err = _map(data, "ont_pi85", ["--align", "--alignMaxLen", str(limit)], ".max")
    n_long = 0
    for a, b, n in zip(got.splitlines(), want.splitlines(), lens):
        if n > limit:
            assert a == AN.strip_tags(b + "\n")[:-1]
            n_long += 1
        else:
            assert a == b
    assert len(got.splitlines()) == len(lens) and 0 < n_long < len(lens)
    assert f"; {n_long} mappings with a region longer than --alignMaxLen {limit} " in err, err[-2000:]
