"""mashmap-b200 --align --eqx / --cs without a device: the options' refusals, the tag restatement the GPU tests check the
device against (tests/align_tags_data.py) pinned on edlib's paths (or the NW restatement's where edlib is not built),
and the layout of the mm_align_batch_tags result."""
import os
import re
import subprocess

import numpy as np
import pytest

import align_data as AD
import align_nw_data as AN
import align_tags_data as AT
from mashmap_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAP_BIN = os.path.join(ROOT, "mashmap_b200", "mashmap-b200")

needs_checker = pytest.mark.skipif(not AN.oracle_nw_available(), reason="oracle/libalign_nw_oracle.so not built")


def _w(path, text):
    with open(path, "w") as f:
        f.write(text)
    return path


@pytest.mark.parametrize("opt", ["--eqx", "--cs"])
@pytest.mark.parametrize("extra", [[], ["--legacy"]])
def test_tag_options_need_align(tmp_path, opt, extra):
    r = _w(str(tmp_path / "r.fa"), ">r\n" + "ACGT" * 500 + "\n")
    p = subprocess.run([MAP_BIN, "-r", r, "-q", r, opt] + extra, capture_output=True, text=True)
    assert p.returncode == 1, p.stderr
    assert f"{opt} is given without --align" in p.stderr, p.stderr
    assert "minmer windows picked" not in p.stderr, p.stderr


@needs_checker
def test_restatement_agrees_with_the_path_it_formats():
    """300 pairs: the extended CIGAR collapses to the standard one (edlib's own edlibAlignmentToCigar(STANDARD) where
    edlib is built), its X + I + D is the distance, cs applied to the target gives the query, and every run is maximal"""
    rng = np.random.default_rng(6060)
    n_n = 0
    for i, (q, t) in enumerate(AT.tag_pairs(rng, 300)):
        ed, ops, std = AT.edlib_or_oracle(q, t)
        assert ed >= 0 and len(ops) > 0, i
        eqx = AT.cigar_eqx(ops)
        assert AT.cigar_std(ops) == std == AT.collapse(eqx), i
        assert AT.eqx_differences(eqx) == ed, i
        assert not re.search(r"([=XID])[0-9]+\1", eqx), i  # adjacent runs differ
        cs = AT.cs_short(ops, q, t)
        assert AT.apply_cs(cs, t) == AT.lower(q), i
        assert AT.cs_differences(cs) == ed, i
        n_n += b"n" in AT.lower(q) and b"n" in AT.lower(t)
    assert n_n >= 50


def test_restatement_examples():
    q, t = np.frombuffer(b"ACGTTNA", dtype=np.uint8), np.frombuffer(b"ACCTNAG", dtype=np.uint8)
    ops = np.array([0, 0, 3, 0, 1, 0, 0, 2], dtype=np.uint8)  # AC G/C T +T N A -G
    assert AT.cigar_std(ops) == "4M1I2M1D"
    assert AT.cigar_eqx(ops) == "2=1X1=1I2=1D"
    assert AT.cs_short(ops, q, t) == ":2*cg:1+t:2-g"
    assert AT.apply_cs(":2*cg:1+t:2-g", t) == b"acgttna"
    assert AT.cs_short(np.array([3, 3], dtype=np.uint8), b"AC", b"GT") == "*ga*tc"


def test_tag_result_layout():
    d = capi.align_tag_result_dtype
    assert d.itemsize == 40
    assert [(n, d.fields[n][0].str, d.fields[n][1]) for n in d.names] == [
        ("ed", "<i4", 0), ("alignment_length", "<i4", 4), ("cg_offset", "<u8", 8), ("cg_len", "<u8", 16),
        ("cs_offset", "<u8", 24), ("cs_len", "<u8", 32)]
    hdr = open(os.path.join(ROOT, "include", "mashmap_b200_align.h")).read()
    body = re.search(r"typedef struct mm_align_tag_result \{(.*?)\} mm_align_tag_result;", hdr, re.S).group(1)
    assert re.findall(r"(\w+)\s+(\w+);", body) == [("int32_t", "ed"), ("int32_t", "alignment_length"),
                                                   ("uint64_t", "cg_offset"), ("uint64_t", "cg_len"),
                                                   ("uint64_t", "cs_offset"), ("uint64_t", "cs_len")]
    flags = {k: 1 << int(v) for k, v in re.findall(r"#define (MM_ALIGN_TAG_\w+) \(1u << (\d+)\)", hdr)}
    assert flags == {"MM_ALIGN_TAG_EQX": capi.MM_ALIGN_TAG_EQX, "MM_ALIGN_TAG_CS": capi.MM_ALIGN_TAG_CS} == {
        "MM_ALIGN_TAG_EQX": 1, "MM_ALIGN_TAG_CS": 2}
    sig = re.search(r"int mm_align_batch_tags\((.*?)\);", hdr, re.S).group(1)
    assert [p.split()[-1].lstrip("*") for p in sig.split(",")] == [
        "ctx", "qbases", "n_qbases", "tbases", "n_tbases", "jobs", "n_jobs", "flags", "results", "text", "text_cap",
        "n_text"]
