"""BGZF input on the GPU: mm_inflate_blocks against zlib, its error reports, and the CLI's PAF on BGZF reference and
queries, byte-identical to plain FASTA and to the line reader (MM_SERIAL_INPUT=1)."""
import gzip
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bgzf_data as B  # noqa: E402
import datasets  # noqa: E402
from conftest import have_gpu  # noqa: E402
from mashmap_b200 import capi, hostlib  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_gpu(), reason="no GPU")]


def _blocks(items):
    comp = b"".join(c for _, c, _ in items)
    coff = np.zeros(len(items) + 1, dtype=np.uint64)
    coff[1:] = np.cumsum([len(c) for _, c, _ in items])
    ooff = np.zeros(len(items) + 1, dtype=np.uint64)
    ooff[1:] = np.cumsum([len(t) for _, _, t in items])
    crc = np.array([zlib.crc32(t) for _, _, t in items], dtype=np.uint32)
    return np.frombuffer(comp, dtype=np.uint8).copy(), coff, ooff, crc


def test_device_inflate_equals_zlib_on_thousands_of_blocks():
    items = B.corpus(seed=1, scale=45)
    assert len(items) > 3000
    inf = capi.Inflater(0)
    comp, coff, ooff, crc = _blocks(items)
    rc, bad, out, err = inf.inflate(comp, coff, ooff, crc)
    assert rc == 0 and bad == -1, err
    assert out[: int(ooff[-1])].tobytes() == b"".join(t for _, _, t in items)
    inf.close()


def test_bad_blocks_are_reported_by_index_and_the_inflater_stays_usable():
    items = B.corpus(seed=2, scale=5)
    inf = capi.Inflater(0)
    comp, coff, ooff, crc = _blocks(items)
    want = b"".join(t for _, _, t in items)
    k = 123
    bad_crc = crc.copy()
    bad_crc[k] ^= 1
    rc, bad, _, err = inf.inflate(comp, coff, ooff, bad_crc)
    assert rc == capi.MM_EINVAL and bad == k and "CRC" in err
    bad_isize = ooff.copy()
    bad_isize[k + 1:] += 1  # block k's output range one byte longer than its text
    rc, bad, _, err = inf.inflate(comp, coff, bad_isize, crc)
    assert rc == capi.MM_EINVAL and bad == k, err
    nonempty = [i for i in range(len(items)) if coff[i + 1] - coff[i] > 8 and len(items[i][2]) > 1000]
    j = nonempty[len(nonempty) // 2]
    bad_stream = comp.copy()
    bad_stream[int(coff[j]):int(coff[j + 1])] = 0xFF  # all-ones: block type 3
    rc, bad, _, err = inf.inflate(bad_stream, coff, ooff, crc)
    assert rc == capi.MM_EINVAL and bad == j, err
    rc, bad, out, err = inf.inflate(comp, coff, ooff, crc)
    assert rc == 0 and bad == -1 and out[: len(want)].tobytes() == want, err
    inf.close()


def _run(cmd, env=None, ok=True):
    p = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    if ok:
        assert p.returncode == 0, (cmd, p.stderr[-2000:])
    return p


def _bgzf_copy(path):
    out = path + ".bgz.gz"
    if not os.path.exists(out):
        B.write_bgzf(out, open(path, "rb").read())
    return out


SETS = {"random": ("bgr", datasets.make_random_set), "panel": ("bgp", datasets.make_panel_set)}
LINES = [
    ("default", "random", ["-s", "5000", "--pi", "85"]),
    ("Y", "panel", ["-s", "5000", "--pi", "95", "-n", "1", "-Y", "#"]),
    ("noSplit", "random", ["-s", "5000", "--pi", "85", "--noSplit"]),
    ("one_to_one", "panel", ["-s", "3000", "--pi", "90", "-f", "one-to-one"]),
    ("align", "random", ["-s", "5000", "--pi", "85", "--align"]),
    ("shards", "panel", ["-s", "5000", "--pi", "85", "--indexShards", "2"]),
    ("targetPrefix", "panel", ["-s", "5000", "--pi", "85", "--targetPrefix", "strain1"]),
    ("small_batches", "random", ["-s", "5000", "--pi", "85", "--batchBases", "30000"]),
]


@pytest.mark.parametrize("tag,which,args", LINES, ids=[x[0] for x in LINES])
def test_cli_paf_is_identical_on_bgzf_input(workdir, tag, which, args):
    d = SETS[which][1](workdir, tag=SETS[which][0])
    ref_gz, qry_gz = _bgzf_copy(d["ref"]), _bgzf_copy(d["qry"])
    outs = {}
    for mode, (r, q, env) in {"plain": (d["ref"], d["qry"], None), "bgzf": (ref_gz, qry_gz, None),
                              "serial": (ref_gz, qry_gz, {"MM_SERIAL_INPUT": "1"})}.items():
        o = os.path.join(workdir, f"bg_{tag}_{mode}.paf")
        p = _run([hostlib.CLI_PATH, "-r", r, "-q", q, "-t", "8", "-o", o] + args, env)
        outs[mode] = open(o).read()
        if mode == "bgzf":
            assert p.stderr.count("BGZF, inflated on device 0") == 2, p.stderr[-2000:]
            if tag == "small_batches":
                assert "in 1 windows" not in p.stderr
    assert outs["plain"] and outs["plain"] == outs["bgzf"] == outs["serial"]


def test_query_list_mixing_bgzf_gzip_fastq_and_plain(workdir):
    d = datasets.make_random_set(workdir, tag="bgr")
    text = open(d["qry"], "rb").read()
    pieces = text.split(b"\n>")
    recs = [(p if i == 0 else b">" + p).rstrip(b"\n") + b"\n" for i, p in enumerate(pieces)]
    part = [b"".join(recs[i::4]) for i in range(4)]
    files = []
    p0 = os.path.join(workdir, "ql_0.fa.gz")
    B.write_bgzf(p0, part[0], block=5000)
    p1 = os.path.join(workdir, "ql_1.fa.gz")
    with open(p1, "wb") as f:
        f.write(gzip.compress(part[1]))
    p2 = os.path.join(workdir, "ql_2.fq")
    with open(p2, "wb") as f:
        for r in part[2].split(b">")[1:]:
            head, _, seq = r.partition(b"\n")
            seq = seq.replace(b"\n", b"")
            f.write(b"@" + head + b"\n" + seq + b"\n+\n" + b"I" * len(seq) + b"\n")
    p3 = os.path.join(workdir, "ql_3.fa")
    with open(p3, "wb") as f:
        f.write(part[3])
    files = [p0, p1, p2, p3]
    ql = os.path.join(workdir, "ql.txt")
    with open(ql, "w") as f:
        f.write("\n".join(files) + "\n")
    outs = []
    for env in (None, {"MM_SERIAL_INPUT": "1"}):
        o = os.path.join(workdir, f"ql_{len(outs)}.paf")
        _run([hostlib.CLI_PATH, "-r", _bgzf_copy(d["ref"]), "--ql", ql, "-s", "5000", "--pi", "85", "-t", "8", "-o", o], env)
        outs.append(open(o).read())
    assert outs[0] and outs[0] == outs[1]


def test_a_corrupt_block_stops_the_cli_naming_its_offset(workdir):
    d = datasets.make_random_set(workdir, tag="bgr")
    blob = bytearray(open(_bgzf_copy(d["qry"]), "rb").read())
    spans = B.member_spans(bytes(blob))
    k = len(spans) // 2
    blob[spans[k][0] + 40] ^= 0x55
    bad = os.path.join(workdir, "corrupt.fa.gz")
    with open(bad, "wb") as f:
        f.write(bytes(blob))
    for r, q in ((d["ref"], bad), (bad, d["qry"])):
        p = _run([hostlib.CLI_PATH, "-r", r, "-q", q, "-s", "5000", "--pi", "85", "-o", os.path.join(workdir, "c.paf")], ok=False)
        assert p.returncode == 1, p.stderr[-2000:]
        assert f"{bad}: corrupt gzip/BGZF block at byte offset {spans[k][0]}" in p.stderr, p.stderr[-2000:]
