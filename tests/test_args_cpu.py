"""The product's option parser fills skch::Parameters exactly as the reference's parseandSave does
(reference src/map/include/parseCmdArgs.hpp:257-659: defaults, automatic sketch size from the file size, --dense,
filter modes, chaining / block-length defaults, skip-self when no query is given ...). CPU only. Where the reference is
not built, against the parameters it produced, stored in tests/golden (golden_ref.py)."""
import os

import pytest

import datasets
import golden_ref
import refh
from mashmap_b200 import hostlib

OPTION_SETS = [
    [],
    ["-s", "5000", "--pi", "85"],
    ["-s", "3000", "--pi", "90", "-f", "one-to-one"],
    ["-s", "5000", "--pi", "95", "--dense"],
    ["-s", "2000", "--pi", "80", "-k", "16", "-J", "25", "--noHgFilter"],
    ["-s", "10000", "--pi", "90", "-n", "3", "--noMerge", "-f", "none"],
    ["-s", "5000", "-X", "-Y", "#", "--lowerTriangular"],
    ["-s", "5000", "-c", "20000", "-l", "10000", "--kmerThreshold", "0.1", "--kmerComplexity", "0.5"],
    ["-s", "1000", "--pi", "99", "--hgFilterAniDiff", "0.5", "--hgFilterConf", "99.0", "--filterLengthMismatches"],
    ["-s", "5000", "-M", "--legacy", "--reportPercentage", "--sparsifyMappings", "0.5"],
    ["-s", "5000", "--numMappingsForShortSeq", "4", "-n", "2", "--dropLowMapId"],
]


@pytest.fixture(scope="module")
def d(workdir):
    return datasets.make_panel_set(workdir, tag="args", n_strains=2, chrom_len=40_000)


def reference_parameters(args, d):
    """skch::Parameters of the reference for a command line, field by field (computed, or stored)"""
    key = golden_ref.key_of(args, d)
    if not refh.available():
        return golden_ref.get("parameters", key)
    R = refh.RefSession(args)
    try:
        got = [getattr(R.p, name) for name, _ in refh.OrcParams._fields_]
    finally:
        R.close()
    golden_ref.check_stored("parameters", key, got)
    return got


@pytest.mark.parametrize("opts", OPTION_SETS, ids=lambda o: " ".join(o) or "defaults")
@pytest.mark.parametrize("with_query", [True, False])
def test_parameters_equal_reference(d, opts, with_query):
    args = ["-r", d["ref"]] + (["-q", d["qry"]] if with_query else []) + ["-t", "2"] + opts
    want = reference_parameters(args, d)
    ours = hostlib.HostIndex.from_cli(args)
    p = ours.params_into(refh.OrcParams())
    for (name, _), a in zip(refh.OrcParams._fields_, want):
        b = getattr(p, name)
        assert a == b, (name, a, b, args)
    ours.close()


@pytest.mark.parametrize("size", [2**31 - 1000, 2**31 + 1000, 3_100_000_000, 5_000_000_000, 2**32 + 4096])
def test_reference_size_wraps_like_the_reference(tmp_path, size):
    """map_parameters.hpp:41 keeps referenceSize in an offset_t (int32): for files >= 2 GiB the value wraps and is
    sign-extended into recommendedSketchSize (parseCmdArgs.hpp:304,639), so the automatic sketch size differs from the
    one the formula gives for the true size. The product reproduces that (a sparse file stands in for the FASTA)."""
    f = tmp_path / "big.fa"
    with open(f, "wb") as fh:
        fh.write(b">c\nACGT\n")
        fh.truncate(size)
    args = ["-r", str(f), "-q", str(f), "-s", "5000", "--pi", "85"]
    ours = hostlib.HostIndex.params_from_cli(args)
    p = ours.params_into(refh.OrcParams())
    ours.close()
    assert [p.referenceSize, p.sketchSize] == reference_size_and_sketch(args, size)


def reference_size_and_sketch(args, size):
    if not refh.available():
        return golden_ref.get("reference_size", str(size))
    ref = refh.parse_only(args)
    got = [ref.referenceSize, ref.sketchSize]
    golden_ref.check_stored("reference_size", str(size), got)
    return got
