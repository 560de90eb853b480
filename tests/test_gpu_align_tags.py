"""mashmap-b200 --align --eqx / --cs on the device: mm_align_batch_tags against mm_align_batch's own paths formatted by
the restatement in tests/align_tags_data.py (short, banded, multi-CTA, all-mismatch, all-N and one-base jobs, every
flag), its capacity and argument errors, and the CLI's three tags against plain --align and the FASTA files."""
import os
import subprocess

import numpy as np
import pytest

import align_data as AD
import align_nw_data as AN
import align_tags_data as AT
import datasets
from conftest import have_gpu
from mashmap_b200 import capi, synth

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_gpu(), reason="no GPU")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAP_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200")
EQX, CS = capi.MM_ALIGN_TAG_EQX, capi.MM_ALIGN_TAG_CS


def _jobs(pairs, mode=capi.MM_ALIGN_NW):
    qb = np.concatenate([p[0] for p in pairs])
    tb = np.concatenate([p[1] for p in pairs])
    jobs = np.zeros(len(pairs), dtype=capi.align_job_dtype)
    jobs["q_len"] = [len(p[0]) for p in pairs]
    jobs["t_len"] = [len(p[1]) for p in pairs]
    jobs["q_offset"][1:] = np.cumsum(jobs["q_len"].astype(np.int64))[:-1]
    jobs["t_offset"][1:] = np.cumsum(jobs["t_len"].astype(np.int64))[:-1]
    jobs["k"] = -1
    jobs["mode"] = mode
    return qb, tb, jobs


def _diverged(rng, n, err):
    t = AD._ACGT[rng.integers(0, 4, size=n)].astype(np.uint8)
    return synth.mutate(t, err, rng, ratio=(30, 2, 1)).astype(np.uint8), t


def _batch(rng):
    pairs = AT.tag_pairs(rng, 3000)
    pairs += [_diverged(rng, 40_000, 0.03), _diverged(rng, 70_000, 0.1)]  # banded (>= MM_ALIGN_BAND_MIN_LEN)
    pairs.append(_diverged(rng, 300_000, 0.02))  # runs and text spread over many CTAs
    a = np.full(500, ord("A"), dtype=np.uint8)
    pairs += [(a, np.full(500, ord("C"), dtype=np.uint8)),  # all mismatches
              (np.full(700, ord("N"), dtype=np.uint8), np.full(650, ord("N"), dtype=np.uint8)),  # all N
              (a[:1], a[:1]), (a[:1], np.frombuffer(b"G", dtype=np.uint8).copy()),
              (a[:1], np.frombuffer(b"CGTAC", dtype=np.uint8).copy()), (np.frombuffer(b"CGTAC", dtype=np.uint8).copy(), a[:1])]
    order = rng.permutation(len(pairs))
    return [pairs[i] for i in order]


@pytest.fixture(scope="module")
def batch():
    rng = np.random.default_rng(9191)
    pairs = _batch(rng)
    ctx = capi.AlignContext(0)
    qb, tb, jobs = _jobs(pairs)
    res, ops = ctx.align(qb, tb, jobs)
    paths = [ops[int(r["ops_offset"]) : int(r["ops_offset"]) + int(r["alignment_length"])] for r in res]
    yield dict(ctx=ctx, pairs=pairs, qb=qb, tb=tb, jobs=jobs, res=res, paths=paths)
    ctx.close()


def _text(text, off, n):
    return text[int(off) : int(off) + int(n)].decode("latin1")


@pytest.mark.parametrize("flags", [0, EQX, CS, EQX | CS])
def test_abi_tags_are_the_paths_of_mm_align_batch(batch, flags):
    ctx = batch["ctx"]
    res, text = ctx.align_tags(batch["qb"], batch["tb"], batch["jobs"], flags)
    assert ctx.tag_ms() > 0
    assert np.array_equal(res["ed"], batch["res"]["ed"])
    assert np.array_equal(res["alignment_length"], batch["res"]["alignment_length"])
    for i, ((q, t), ops, r) in enumerate(zip(batch["pairs"], batch["paths"], res)):
        assert len(ops) > 0, i
        want = AT.cigar_eqx(ops) if flags & EQX else AT.cigar_std(ops)
        assert _text(text, r["cg_offset"], r["cg_len"]) == want, (i, len(q), len(t))
        if flags & CS:
            assert _text(text, r["cs_offset"], r["cs_len"]) == AT.cs_short(ops, q, t), (i, len(q), len(t))
        else:
            assert r["cs_len"] == 0
    assert max(len(p[0]) for p in batch["pairs"]) >= 300_000


def test_abi_capacity_reports_the_exact_size(batch):
    ctx = batch["ctx"]
    res, text = ctx.align_tags(batch["qb"], batch["tb"], batch["jobs"], EQX | CS)
    with pytest.raises(capi.MashmapError) as e:
        ctx.align_tags(batch["qb"], batch["tb"], batch["jobs"], EQX | CS, text_cap=len(text) - 1)
    assert e.value.code == capi.MM_ECAPACITY and e.value.n_text == len(text)
    res2, text2 = ctx.align_tags(batch["qb"], batch["tb"], batch["jobs"], EQX | CS, text_cap=len(text))
    assert text2 == text and np.array_equal(res2, res)


def test_abi_refuses_hw_jobs_and_unknown_flags():
    ctx = capi.AlignContext(0)
    q = np.frombuffer(b"ACGTACGTAC", dtype=np.uint8)
    jobs = np.zeros(2, dtype=capi.align_job_dtype)
    jobs["q_len"], jobs["t_len"], jobs["k"], jobs["mode"] = 10, 10, -1, capi.MM_ALIGN_NW
    jobs["mode"][1] = capi.MM_ALIGN_HW
    with pytest.raises(capi.MashmapError) as e:
        ctx.align_tags(q, q, jobs)
    assert e.value.code == capi.MM_EINVAL and "MM_ALIGN_NW" in str(e.value)
    with pytest.raises(capi.MashmapError) as e:
        ctx.align_tags(q, q, jobs[:1], flags=4)
    assert e.value.code == capi.MM_EINVAL and "flags" in str(e.value)
    res, text = ctx.align_tags(q, q, jobs[:1], EQX | CS)
    assert text == b"10=:10" and res["cg_len"][0] == 3 and res["cs_offset"][0] == 3
    ctx.close()


# ---- the CLI ---------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("align_tags"))
    rnd = datasets.make_random_set(d, tag="at", n_contigs=3, contig_len=300_000, n_reads=40, read_len=10_000, seed=71)
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
    "ont_nosplit": ("rnd", ["--pi", "85", "--noSplit"]),
    "asm_one_to_one": ("asm", ["--pi", "90", "-s", "2000", "-f", "one-to-one"]),
}
_runs = {}


def _map(data, name, extra=()):
    key = (name, tuple(extra))
    if key not in _runs:
        which, opts = CASES[name]
        ref, qry = (data["ref"], data["qry"]) if which == "rnd" else (data["asm_ref"], data["asm_qry"])
        out = os.path.join(data["dir"], f"{name}.{len(_runs)}.paf")
        p = subprocess.run([MAP_BIN, "-r", ref, "-q", qry, "-o", out] + opts + list(extra), capture_output=True,
                           text=True, cwd=data["dir"])
        assert p.returncode == 0, p.stderr[-3000:]
        _runs[key] = (open(out).read(), p.stderr)
    return _runs[key]


def _fasta(data, name):
    which = CASES[name][0]
    fa = (data["qry"], data["ref"]) if which == "rnd" else (data["asm_qry"], data["asm_ref"])
    return AN.read_fasta(fa[0]), AN.read_fasta(fa[1])


TAGS = ["--align", "--eqx", "--cs"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_cli_tags_agree_with_plain_align_and_the_sequences(data, name):
    plain, err_plain = _map(data, name, ["--align"])
    text, err = _map(data, name, TAGS)
    tagged, untagged = AT.check_tag_paf(text, plain, *_fasta(data, name))
    assert tagged == plain.count("\n") > 5 and untagged == 0
    assert f"] {tagged} mappings aligned" in err and f"] {tagged} mappings aligned" in err_plain
    assert {ln.split("\t")[4] for ln in text.splitlines()} == {"+", "-"}
    assert any("*" in ln.split("\t")[-1] and "+" in ln.split("\t")[-1] for ln in text.splitlines())


def test_cli_each_option_alone(data):
    plain, _ = _map(data, "asm_one_to_one", ["--align"])
    both, _ = _map(data, "asm_one_to_one", TAGS)
    eqx, _ = _map(data, "asm_one_to_one", ["--align", "--eqx"])
    cs, _ = _map(data, "asm_one_to_one", ["--align", "--cs"])
    assert eqx == "".join(ln.rsplit("\t", 1)[0] + "\n" for ln in both.splitlines())
    for a, b, c in zip(cs.splitlines(), plain.splitlines(), both.splitlines()):
        assert a == b + "\t" + c.rsplit("\t", 1)[1]


def test_cli_align_max_len_drops_all_three_tags(data):
    plain, _ = _map(data, "ont_pi85", ["--align"])
    lens = [max(int(f[3]) - int(f[2]), int(f[8]) - int(f[7])) for f in (ln.split("\t") for ln in plain.splitlines())]
    limit = sorted(lens)[len(lens) // 2]
    plain_max, _ = _map(data, "ont_pi85", ["--align", "--alignMaxLen", str(limit)])
    text, _ = _map(data, "ont_pi85", TAGS + ["--alignMaxLen", str(limit)])
    tagged, untagged = AT.check_tag_paf(text, plain_max, *_fasta(data, "ont_pi85"), max_len=limit)
    assert tagged > 0 and untagged == sum(n > limit for n in lens) > 0


@pytest.mark.parametrize("name", ["ont_pi85", "asm_one_to_one"])
def test_cli_output_does_not_depend_on_batches_or_threads(data, name):
    want, _ = _map(data, name, TAGS)
    for extra in (["--batchBases", "30000", "--subBatchBases", "12000", "-t", "1"], ["-t", "8"]):
        got, _ = _map(data, name, TAGS + extra)
        assert got == want, extra


def _gpu_count():
    import torch

    return torch.cuda.device_count() if have_gpu() else 0


@pytest.mark.skipif(_gpu_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("name", ["ont_pi85", "asm_one_to_one"])
def test_cli_output_does_not_depend_on_devices(data, name):
    want, _ = _map(data, name, TAGS)
    got, _ = _map(data, name, TAGS + ["--devices", "0,1", "--subBatchBases", "30000"])
    assert got == want
