"""FASTQ parsed on the GPU: mm_fastq_cut against the host build of the same cut (mashmap_b200/csrc/mm_fastq.h) and
against a plain statement of the records, and the CLI's PAF on FASTQ queries, plain and BGZF, byte-identical to the
same reads as FASTA and to the line reader (MM_SERIAL_INPUT=1)."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bgzf_data as B  # noqa: E402
import datasets  # noqa: E402
import fastq_data as Q  # noqa: E402
from conftest import have_gpu  # noqa: E402
from mashmap_b200 import capi, hostlib  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_gpu(), reason="no GPU")]

WINDOWS = [1, 7, 100, 4096, 65536, 1 << 20]


def _write(path, blob):
    with open(path, "wb") as f:
        f.write(blob)
    return str(path)


def _n_gpus():
    try:
        import torch

        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("window", WINDOWS)
def test_device_cut_equals_the_host_build_and_the_line_reader(tmp_path, window):
    for name, text in Q.awkward(seed=window).items():
        files = {"plain": _write(tmp_path / f"{name}.fq", text),
                 "bgzf": _write(tmp_path / f"{name}.fq.gz", B.bgzf(text, block=777))}
        for kind, p in files.items():
            want = hostlib.fastq_digest(p)
            host = hostlib.fastq_digest(p, window, threads=2)
            dev = hostlib.fastq_digest(p, window, threads=2, device=0)
            assert dev == host and dev[:3] == want[:3], (name, kind, window, dev, host, want)


def _records(text):
    """(names, sequences) of a FASTQ text without empty header lines, four lines per record"""
    lines = text.split(b"\n")
    return [lines[i][1:].split(b" ")[0] for i in range(0, len(lines) - 1, 4)], [lines[i + 1] for i in range(0, len(lines) - 1, 4)]


def _check_window(fq, text, last=1):
    fq.append_text(text)
    got = fq.cut(last)
    names, seqs = _records(text)
    assert got["ended"] == 0 and got["consumed"] == len(text)
    assert got["names"] == names
    assert [int(x) for x in got["seq_len"]] == [len(s) for s in seqs]
    want = b"".join(capi.pack_bases(np.frombuffer(s, dtype=np.uint8)).tobytes() for s in seqs)
    assert got["nib_all"] == want
    return got


def test_a_window_of_over_a_million_records():
    rng = np.random.default_rng(5)
    n = 1_100_000
    lens = rng.integers(0, 40, n)
    bases = B.dna(rng, int(lens.sum()))
    out, o = [], 0
    for i, ln in enumerate(lens.tolist()):
        out.append(b"@q%d x\n%s\n+\n%s\n" % (i, bases[o:o + ln], b"I" * ln))
        o += ln
    fq = capi.FastqParser(0)
    got = _check_window(fq, b"".join(out))
    assert len(got["names"]) == n
    fq.close()


def test_ultra_long_reads_beside_short_ones():
    rng = np.random.default_rng(6)
    parts = []
    for i in range(400):
        ln = 1_000_000 + i if i % 100 == 7 else int(rng.integers(90, 111))
        s = Q.dna(rng, ln, Q.IUPAC)
        parts.append(b"@r%d\n%s\n+\n%s\n" % (i, s, b"#" * ln))
    fq = capi.FastqParser(0)
    _check_window(fq, b"".join(parts))
    # the same text over many appends and cuts: records come out in order, each exactly once
    text = b"".join(parts)
    names, seqs = [], []
    for o in range(0, len(text), 300_000):
        fq.append_text(text[o:o + 300_000])
        got = fq.cut(1 if o + 300_000 >= len(text) else 0)
        names += got["names"]
        seqs += [int(x) for x in got["seq_len"]]
    want_names, want_seqs = _records(text)
    assert names == want_names and seqs == [len(s) for s in want_seqs]
    ms = fq.last_ms()
    assert ms[1] >= ms[0] > 0
    fq.close()


def test_bgzf_blocks_inflate_into_the_window_and_bad_ones_are_reported():
    rng = np.random.default_rng(7)
    text = Q.fastq(rng, 300, [100, 5000])
    items = [(None, B.deflate_raw(text[o:o + 20000]), text[o:o + 20000]) for o in range(0, len(text), 20000)]
    import zlib

    comp = np.frombuffer(b"".join(c for _, c, _ in items), dtype=np.uint8)
    coff = np.concatenate([[0], np.cumsum([len(c) for _, c, _ in items])]).astype(np.uint64)
    ooff = np.concatenate([[0], np.cumsum([len(t) for _, _, t in items])]).astype(np.uint64)
    crc = np.array([zlib.crc32(t) for _, _, t in items], dtype=np.uint32)
    fq = capi.FastqParser(0)
    bad_crc = crc.copy()
    bad_crc[3] ^= 1
    rc, bad, err = fq.append_blocks(comp, coff, ooff, bad_crc)
    assert rc == capi.MM_EINVAL and bad == 3 and "CRC" in err
    fq.close()
    fq = capi.FastqParser(0)
    rc, bad, err = fq.append_blocks(comp, coff, ooff, crc)
    assert rc == 0 and bad == -1, err
    got = fq.cut(1)
    names, seqs = _records(text)
    assert got["names"] == names and [int(x) for x in got["seq_len"]] == [len(s) for s in seqs]
    fq.close()


def _run(cmd, env=None, ok=True):
    p = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    if ok:
        assert p.returncode == 0, (cmd, p.stderr[-2000:])
    return p


def _as_fastq(fasta_path, out):
    """the records of a FASTA file as FASTQ (one sequence line, a quality line of the same length)"""
    if not os.path.exists(out):
        text = open(fasta_path, "rb").read()
        with open(out, "wb") as f:
            for r in text.split(b">")[1:]:
                head, _, seq = r.partition(b"\n")
                seq = seq.replace(b"\n", b"")
                f.write(b"@" + head + b"\n" + seq + b"\n+\n" + b"5" * len(seq) + b"\n")
    return out


LINES = [
    ("default", ["-s", "5000", "--pi", "85"]),
    ("t1", ["-s", "5000", "--pi", "85", "-t", "1"]),
    ("small_batches", ["-s", "5000", "--pi", "85", "--batchBases", "30000"]),
    ("one_to_one", ["-s", "3000", "--pi", "90", "-f", "one-to-one"]),
    ("align", ["-s", "5000", "--pi", "85", "--align"]),
    ("noSplit", ["-s", "5000", "--pi", "85", "--noSplit"]),
]


@pytest.mark.parametrize("tag,args", LINES, ids=[x[0] for x in LINES])
def test_cli_paf_is_identical_on_fastq_queries(workdir, tag, args):
    d = datasets.make_random_set(workdir, tag="fqr")
    fq = _as_fastq(d["qry"], os.path.join(workdir, "fqr_reads.fq"))
    fq_gz = fq + ".gz"
    if not os.path.exists(fq_gz):
        B.write_bgzf(fq_gz, open(fq, "rb").read())
    threads = [] if "-t" in args else ["-t", "8"]
    outs = {}
    for mode, (q, env) in {"fasta": (d["qry"], None), "fastq": (fq, None), "bgzf": (fq_gz, None),
                           "serial": (fq, {"MM_SERIAL_INPUT": "1"})}.items():
        o = os.path.join(workdir, f"fq_{tag}_{mode}.paf")
        p = _run([hostlib.CLI_PATH, "-r", d["ref"], "-q", q, "-o", o] + threads + args, env)
        outs[mode] = open(o).read()
        if mode in ("fastq", "bgzf"):
            assert f"{q}: FASTQ, parsed on device 0 in" in p.stderr, p.stderr[-2000:]
            if tag == "small_batches":
                assert " in 1 windows" not in p.stderr
        if mode == "serial":
            assert "FASTQ, parsed on device" not in p.stderr
    assert outs["fasta"] and outs["fasta"] == outs["fastq"] == outs["bgzf"] == outs["serial"]


def test_query_list_mixing_fastq_bgzf_fastq_and_fasta(workdir):
    d = datasets.make_random_set(workdir, tag="fqr")
    text = open(d["qry"], "rb").read()
    recs = [b">" + r for r in text.split(b">")[1:]]
    part = [b"".join(recs[i::3]) for i in range(3)]
    p0 = _write(os.path.join(workdir, "fql_0.fa"), part[0])
    p1 = _as_fastq(_write(os.path.join(workdir, "fql_1.fa"), part[1]), os.path.join(workdir, "fql_1.fq"))
    p2 = os.path.join(workdir, "fql_2.fq.gz")
    B.write_bgzf(p2, open(_as_fastq(_write(os.path.join(workdir, "fql_2.fa"), part[2]), os.path.join(workdir, "fql_2.fq")), "rb").read(), block=3000)
    ql = _write(os.path.join(workdir, "fql.txt"), "\n".join([p1, p0, p2]).encode() + b"\n")
    outs = []
    for env in (None, {"MM_SERIAL_INPUT": "1"}):
        o = os.path.join(workdir, f"fql_{len(outs)}.paf")
        _run([hostlib.CLI_PATH, "-r", d["ref"], "--ql", ql, "-s", "5000", "--pi", "85", "-t", "8", "-o", o], env)
        outs.append(open(o).read())
    assert outs[0] and outs[0] == outs[1]


@pytest.mark.skipif(_n_gpus() < 2, reason="needs two GPUs")
def test_two_devices_give_the_same_paf(workdir):
    d = datasets.make_random_set(workdir, tag="fqr")
    fq = _as_fastq(d["qry"], os.path.join(workdir, "fqr_reads.fq"))
    outs = []
    for dev in (["--device", "0"], ["--devices", "0-1"]):
        o = os.path.join(workdir, f"fq_dev_{len(outs)}.paf")
        _run([hostlib.CLI_PATH, "-r", d["ref"], "-q", fq, "-s", "5000", "--pi", "85", "-o", o] + dev)
        outs.append(open(o).read())
    assert outs[0] and outs[0] == outs[1]


def test_a_corrupt_member_stops_the_cli_naming_its_offset(workdir):
    d = datasets.make_random_set(workdir, tag="fqr")
    fq = _as_fastq(d["qry"], os.path.join(workdir, "fqr_reads.fq"))
    blob = bytearray(B.bgzf(open(fq, "rb").read()))
    spans = B.member_spans(bytes(blob))
    k = len(spans) // 2
    blob[spans[k][0] + 40] ^= 0x55
    bad = _write(os.path.join(workdir, "corrupt.fq.gz"), bytes(blob))
    p = _run([hostlib.CLI_PATH, "-r", d["ref"], "-q", bad, "-s", "5000", "--pi", "85", "-o", os.path.join(workdir, "c.paf")], ok=False)
    assert p.returncode == 1, p.stderr[-2000:]
    assert f"{bad}: corrupt gzip/BGZF block at byte offset {spans[k][0]}" in p.stderr, p.stderr[-2000:]
