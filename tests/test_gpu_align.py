"""mashmap-b200-align on the device: its output file byte for byte against the unmodified reference aligner
(oracle/_ref/mashmap_align_ref, or the sha256 of its output stored in tests/golden/align/ where it is not built), and the
C ABI per pair against edlib (oracle/_ref/libedlib_ref.so, or the full-matrix restatement oracle/libalign_oracle.so)."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import align_cases as AC
import align_data as AD
from mashmap_b200 import capi

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALIGN_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200-align")
MAP_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200")


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    return AC.write_inputs(str(tmp_path_factory.mktemp("align")))


def _expected(d, name):
    """(sha256, text or None) of the reference aligner's output for a case"""
    if os.path.exists(AD.ALIGN_REF_BIN):
        o = os.path.join(d, name + ".ref.sam")
        subprocess.run([AD.ALIGN_REF_BIN] + AC.case_args(d, name) + ["-o", o], check=True, capture_output=True, cwd=d)
        data = open(o, "rb").read()
        return hashlib.sha256(data).hexdigest(), data
    golden = json.load(open(os.path.join(AC.GOLDEN, "reference_outputs.json")))
    return golden[name]["sha256"], None


def _run(d, name, extra=()):
    o = os.path.join(d, name + ".b200.sam")
    p = subprocess.run([ALIGN_BIN] + AC.case_args(d, name) + ["-o", o] + list(extra), capture_output=True, text=True, cwd=d)
    assert p.returncode == 0, p.stderr
    return open(o, "rb").read()


def test_mapper_legacy_output_is_the_stored_mapping_file(inputs):
    """the mapping file the ONT cases align is what `mashmap-b200 --legacy` prints for these inputs"""
    out = os.path.join(inputs, "legacy.map")
    p = subprocess.run([MAP_BIN, "-r", os.path.join(inputs, "ref.fa"), "-q", os.path.join(inputs, "reads.fa"), "--pi", "80",
                        "--legacy", "-o", out], capture_output=True, text=True, cwd=inputs)
    assert p.returncode == 0, p.stderr
    assert open(out, "rb").read() == open(AC.MAPPED, "rb").read()


@pytest.mark.parametrize("name", sorted(AC.CASES))
def test_output_byte_identical_to_reference_aligner(inputs, name):
    want_sha, want = _expected(inputs, name)
    got = _run(inputs, name)
    if want is not None:
        assert got == want
    assert hashlib.sha256(got).hexdigest() == want_sha


def test_tiny_batches_give_the_same_output(inputs):
    """--batchBases smaller than one mapping: one device batch per mapping line"""
    want_sha, _ = _expected(inputs, "ont_pi80")
    got = _run(inputs, "ont_pi80", ["--batchBases", "1000"])
    assert hashlib.sha256(got).hexdigest() == want_sha


def test_abi_matches_edlib_on_random_pairs():
    """>= 50,000 pairs of the CPU test's generator through mm_align_batch, in a few batches"""
    rng = np.random.default_rng(2024)
    use_ref = AD.edlib_ref_available()
    check = AD.edlib_ref_align if use_ref else AD.oracle_align
    ctx = capi.AlignContext(0)
    total = 0
    for batch in range(5):
        pairs = []
        for i in range(10_400):
            q, t = AD.random_pair(rng) if i % 200 else AD.threshold_pair(rng)
            r = rng.random()
            k = -1 if r < 0.3 else (len(q) if r < 0.5 else int(rng.integers(0, max(1, len(q) // 2))))
            pairs.append((q, t, k))
        qb = np.concatenate([p[0] for p in pairs])
        tb = np.concatenate([p[1] for p in pairs])
        jobs = np.zeros(len(pairs), dtype=capi.align_job_dtype)
        jobs["q_len"] = [len(p[0]) for p in pairs]
        jobs["t_len"] = [len(p[1]) for p in pairs]
        jobs["q_offset"][1:] = np.cumsum(jobs["q_len"].astype(np.int64))[:-1]
        jobs["t_offset"][1:] = np.cumsum(jobs["t_len"].astype(np.int64))[:-1]
        jobs["k"] = [p[2] for p in pairs]
        res, ops = ctx.align(qb, tb, jobs)
        for i, (q, t, k) in enumerate(pairs):
            want = check(q, t, k)
            r = res[i]
            o = int(r["ops_offset"])
            got_ops = ops[o : o + int(r["alignment_length"])]
            assert (int(r["ed"]), int(r["start"]), int(r["end"])) == tuple(want[:3]), (batch, i, len(q), len(t), k)
            assert np.array_equal(got_ops, want[3]), (batch, i, len(q), len(t), k)
        total += len(pairs)
    assert total >= 50_000
    ctx.close()


def test_abi_capacity_error_reports_the_needed_size():
    ctx = capi.AlignContext(0)
    q = np.frombuffer(b"ACGTACGTAC", dtype=np.uint8)
    jobs = np.zeros(1, dtype=capi.align_job_dtype)
    jobs["q_len"], jobs["t_len"], jobs["k"] = 10, 10, -1
    with pytest.raises(capi.MashmapError) as e:
        ctx.align(q, q, jobs, ops_cap=3)
    assert e.value.code == capi.MM_ECAPACITY and e.value.n_ops == 10
    res, ops = ctx.align(q, q, jobs)
    assert res[0]["ed"] == 0 and res[0]["alignment_length"] == 10 and not ops.any()
    ctx.close()
