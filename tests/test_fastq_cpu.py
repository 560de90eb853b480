"""The FASTQ window reader without a GPU: the host build of the cut (mashmap_b200/csrc/mm_fastq.h), fed windows from one
byte up, gives the line reader's records -- names, lengths, nibbles and their count -- on awkward files, plain and
BGZF; and the line reader agrees with the reference's own reader on them."""
import ctypes as C
import gzip
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bgzf_data as B  # noqa: E402
import fastq_data as Q  # noqa: E402
from mashmap_b200 import hostlib  # noqa: E402

WINDOWS = [1, 7, 100, 4096, 65536, 1 << 20]


def _write(path, blob):
    with open(path, "wb") as f:
        f.write(blob)
    return str(path)


def _line_reader_records(text):
    """the line reader's record count, restated: four lines per record, an empty header line ends the file"""
    lines = text.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    n = 0
    for i in range(0, len(lines), 4):
        if lines[i] == b"" and i:
            break
        n += 1
    return n


@pytest.mark.parametrize("window", WINDOWS)
def test_host_cut_equals_the_line_reader_on_plain_fastq(tmp_path, window):
    for name, text in Q.awkward(seed=window).items():
        p = _write(tmp_path / f"{name}.fq", text)
        want = hostlib.fastq_digest(p)
        assert want[0] == _line_reader_records(text), name
        got = hostlib.fastq_digest(p, window, threads=3)
        assert got[:3] == want[:3], (name, window, got, want)
        if name == "plain" and window <= 100:
            assert got[3] > 3


@pytest.mark.parametrize("window", WINDOWS)
def test_host_cut_equals_the_line_reader_on_bgzf_fastq(tmp_path, window):
    for name, text in Q.awkward(seed=window + 1).items():
        half = len(text) // 2
        blobs = {
            "bgzf": B.bgzf(text, block=777),
            "mixed": B.bgzf(text[:half], block=1000, eof=False) + gzip.compress(text[half:half + 500], mtime=0)
                     + B.bgzf(text[half + 500:], block=333),
            "truncated_last": B.bgzf(text, block=min(B.BLOCK, len(text) // 3 + 1), eof=False)[:-3],
            "garbage_tail": B.bgzf(text, block=5000) + b"not gzip at all" * 3,
        }
        for kind, blob in blobs.items():
            p = _write(tmp_path / f"{name}_{kind}.fq.gz", blob)
            want = hostlib.fastq_digest(p)
            got = hostlib.fastq_digest(p, window, threads=2)
            assert got[:3] == want[:3], (name, kind, window, got, want)


def test_the_window_reader_takes_only_fastq(tmp_path):
    fq = b"@r1\nACGT\n+\nIIII\n"
    cases = {"fasta": b">r1\nACGT\n", "gzip_fastq": gzip.compress(fq), "bgzf_fasta": B.bgzf(b">r1\nACGT\n"), "empty": b"",
             "text": b"hello\n"}
    for name, blob in cases.items():
        assert hostlib.fastq_digest(_write(tmp_path / name, blob), 4096) is None, name
    assert hostlib.fastq_digest(_write(tmp_path / "p.fq", fq), 4096)[0] == 1
    assert hostlib.fastq_digest(_write(tmp_path / "b.fq.gz", B.bgzf(fq)), 4096)[0] == 1
    # the FASTA readers keep declining FASTQ
    assert hostlib.fasta_readers_diff(str(tmp_path / "p.fq"))[0] == -1
    assert hostlib.bgzf_text(str(tmp_path / "b.fq.gz"))[0] is None


def test_a_corrupt_member_names_the_file_and_its_offset(tmp_path):
    rng = np.random.default_rng(4)
    text = Q.fastq(rng, 200, [3000])
    blob = bytearray(B.bgzf(text, block=10000))
    spans = B.member_spans(bytes(blob))
    k = len(spans) // 2
    blob[spans[k][0] + 30] ^= 0x10
    p = _write(tmp_path / "bad.fq.gz", bytes(blob))
    with pytest.raises(RuntimeError, match=f"{p}: corrupt gzip/BGZF block at byte offset {spans[k][0]}:"):
        hostlib.fastq_digest(p, 1 << 16)


def test_the_line_reader_equals_the_reference_reader_on_the_same_files(tmp_path):
    import refh

    if not refh.available():
        pytest.skip("oracle/_ref/libmm_ref.so not built")
    R, H = refh.lib(), hostlib.lib()
    R.refh_read_file_digest.argtypes = [C.c_char_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    for name, text in Q.awkward(seed=3).items():
        if name.startswith("empty_header") or name == "cut_after_1":
            # the reference throws on an empty header line, and loops on in.good(), so it drops a last header line
            # that has no '\n'; the line reader keeps that record, and the window reader follows the line reader
            continue
        for kind, blob in (("plain", text), ("bgzf", B.bgzf(text, block=999))):
            p = _write(tmp_path / f"{name}_{kind}.fq", blob)
            want = [C.c_uint64() for _ in range(3)]
            assert R.refh_read_file_digest(p.encode(), *[C.byref(x) for x in want]) == 0, name
            got = [C.c_uint64() for _ in range(3)]
            assert H.skch_read_file_digest(p.encode(), 0, 1, *[C.byref(x) for x in got]) == 0
            assert [x.value for x in got] == [x.value for x in want], (name, kind)
            # ... and the window reader gives the line reader's records (names, lengths, nibbles)
            assert hostlib.fastq_digest(p, 4096)[:3] == hostlib.fastq_digest(p)[:3], (name, kind)
