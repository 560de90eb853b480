"""The BGZF input path without a GPU: the host build of the DEFLATE decoder (mashmap_b200/csrc/mm_inflate.h) against
zlib, its bounds under ASan and UBSan, the member scan against gzread, and the windowed reader against the line reader."""
import ctypes as C
import gzip
import os
import shutil
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bgzf_data as B  # noqa: E402
from mashmap_b200 import hostlib  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_host_decoder_equals_zlib_on_the_corpus():
    corpus = B.corpus(scale=2)
    assert len(corpus) > 100
    for name, comp, text in corpus:
        rc, out, crc = hostlib.mmi_inflate(comp, len(text))
        assert rc == 0, name
        assert out == text, name
        assert crc == zlib.crc32(text), name


def test_host_decoder_rejects_a_wrong_output_size():
    text = b"ACGT" * 5000
    comp = B.deflate_raw(text)
    assert hostlib.mmi_inflate(comp, len(text) - 1)[0] == 2  # MMI_E_OUTPUT
    assert hostlib.mmi_inflate(comp, len(text) + 1)[0] == 3  # MMI_E_SHORT
    assert hostlib.mmi_inflate(comp + b"\0", len(text))[0] == 9  # MMI_E_TRAILING


def _zlib_view(comp, out_len):
    """(accepted, crc) as zlib sees the same stream with the decoder's rules: a complete raw stream on exactly these
    bytes that inflates to out_len bytes"""
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(comp, out_len + 1)
    except zlib.error:
        return False, 0
    ok = d.eof and not d.unused_data and not d.unconsumed_tail and len(out) == out_len
    return ok, (zlib.crc32(out) if ok else 0)


@pytest.mark.skipif(shutil.which("g++") is None, reason="no g++")
def test_malformed_streams_end_in_an_error_within_bounds_under_asan_and_ubsan(tmp_path):
    exe = str(tmp_path / "inflate_cases")
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
           "-fno-omit-frame-pointer", "-I", os.path.join(ROOT, "mashmap_b200", "csrc"),
           os.path.join(ROOT, "tests", "tools", "inflate_cases.cpp"), "-o", exe]
    p = subprocess.run(cmd, capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    rng = np.random.default_rng(3)
    cases = []
    for name, comp, text in B.corpus(seed=9):
        if len(comp) == 0:
            continue
        cases.append((comp, len(text)))
        for _ in range(6):  # bit flips
            b = bytearray(comp)
            for _ in range(int(rng.integers(1, 4))):
                i = int(rng.integers(0, len(b)))
                b[i] ^= 1 << int(rng.integers(0, 8))
            cases.append((bytes(b), len(text)))
        for cut in sorted({1, len(comp) // 2, len(comp) - 1}):  # truncations
            if 0 < cut < len(comp):
                cases.append((comp[:cut], len(text)))
        cases.append((comp, max(0, len(text) - 7)))
        cases.append((rng.integers(0, 256, len(comp), dtype=np.uint8).tobytes(), len(text)))  # noise
    blob = b"".join(struct.pack("<II", len(c), n) + c for c, n in cases)
    path = tmp_path / "cases.bin"
    path.write_bytes(blob)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    p = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env)
    assert p.returncode == 0, p.stderr[-3000:]
    lines = p.stdout.split("\n")[:-1]
    assert len(lines) == len(cases)
    n_err = 0
    for (c, n), line in zip(cases, lines):
        rc, crc = (int(v) for v in line.split())
        ok, zcrc = _zlib_view(c, n)
        assert (rc == 0) == ok, (rc, ok, len(c), n)
        assert crc == zcrc
        n_err += rc != 0
    assert n_err > len(cases) // 3


def _fasta(rng, n_rec, lens, width=60, crlf=False, final_newline=True, blank=False):
    out = []
    for i in range(n_rec):
        s = B.dna(rng, int(rng.choice(lens)))
        out.append(b">rec%d some description\n" % i)
        for o in range(0, len(s), width):
            out.append(s[o : o + width] + b"\n")
        if blank:
            out.append(b"\n")
    t = b"".join(out)
    if crlf:
        t = t.replace(b"\n", b"\r\n")
    if not final_newline:
        t = t.rstrip(b"\r\n")
    return t


def test_member_scan_gives_gzreads_text(tmp_path):
    rng = np.random.default_rng(1)
    a = _fasta(rng, 40, [100, 3000, 70000])
    b = _fasta(rng, 10, [500])
    plain = gzip.compress(b, mtime=0)
    cases = {
        "bgzf": B.bgzf(a),
        "no_eof_marker": B.bgzf(a, eof=False),
        "mixed": B.bgzf(a) + plain + B.bgzf(b, block=999),
        "empty_members": B.EOF_MARKER.join([B.bgzf(a[:5000], eof=False), B.bgzf(a[5000:])]),
        "trailing_garbage": B.bgzf(a) + b"this is not gzip" * 10,
        "trailing_zeros": B.bgzf(a) + b"\0" * 100,
        "truncated_last": B.bgzf(a, eof=False)[:-5000],
        "truncated_trailer": B.bgzf(a, eof=False)[:-3],
        "truncated_plain": B.bgzf(a) + plain[: len(plain) // 2],
        "single_byte_tail": B.bgzf(a) + b"\x1f",
    }
    for name, blob in cases.items():
        p = str(tmp_path / (name + ".fa.gz"))
        with open(p, "wb") as f:
            f.write(blob)
        want = hostlib.gzread_text(p)
        for window in (1, 70000, 1 << 22):
            got, nw, _ = hostlib.bgzf_text(p, window)
            assert got == want, (name, window, len(got or b""), len(want))


def test_files_whose_first_member_is_not_bgzf_are_declined(tmp_path):
    rng = np.random.default_rng(2)
    a = _fasta(rng, 5, [100])
    for name, blob in {"gzip": gzip.compress(a), "gzip_then_bgzf": gzip.compress(a) + B.bgzf(a), "plain": a,
                       "fastq_in_bgzf": B.bgzf(b"@r1\nACGT\n+\nIIII\n")}.items():
        p = str(tmp_path / name)
        with open(p, "wb") as f:
            f.write(blob)
        assert hostlib.bgzf_text(p)[0] is None, name
    assert hostlib.fasta_readers_diff(str(tmp_path / "gzip_then_bgzf"))[0] == -1  # the bulk reader still declines gzip


@pytest.mark.parametrize("window", [1, 100, 4096, 65536, 1 << 20])
def test_windowed_reader_equals_the_line_reader(tmp_path, window):
    rng = np.random.default_rng(window)
    texts = {
        "spanning": _fasta(rng, 200, [0, 1, 59, 60, 61, 900, 5000]),
        "long_record": _fasta(rng, 3, [10, 300000, 20]),
        "crlf_blank": _fasta(rng, 50, [0, 70, 2000], crlf=True, blank=True),
        "no_final_newline": _fasta(rng, 30, [1000], final_newline=False),
        "empty_record_last": _fasta(rng, 20, [500]) + b">empty\n",
        "header_only_no_newline": _fasta(rng, 20, [500]) + b">last",
        "gt_inside": b">a >b\nAC>GT\n>c\n\n>d\nTT\n",
    }
    for name, text in texts.items():
        for block in (B.BLOCK, 777):
            p = B.write_bgzf(tmp_path / f"{name}_{block}.fa.gz", text, block=block)
            d, nr, nb = hostlib.bgzf_readers_diff(p, window, threads=3)
            assert d == 0 and nr == text.count(b"\n>") + 1, (name, block, d, nr)
            got, nw, _ = hostlib.bgzf_text(p, window)
            assert got == text
            if window <= 4096 and name == "spanning":
                assert nw > 3, (name, nw)


def test_a_bad_block_stops_the_reader_and_names_its_offset(tmp_path):
    rng = np.random.default_rng(4)
    text = _fasta(rng, 100, [5000])
    blob = B.bgzf(text, block=10000)
    spans = B.member_spans(blob)
    p = str(tmp_path / "x.fa.gz")
    with open(p, "wb") as f:
        f.write(blob)
    # the inflater's report of block k (a fake that rejects it) comes back as the member's byte offset
    for k in (0, 3, len(spans) - 2):
        with pytest.raises(RuntimeError, match=f"byte offset {spans[k][0]}:"):
            hostlib.bgzf_text(p, 30000, fail_block=k)
    # a flipped bit in a member's data (or its CRC) is found by the decoder
    for k, at in ((2, 30), (5, -6)):
        bad = bytearray(blob)
        bad[spans[k][1] + at if at < 0 else spans[k][0] + at] ^= 0x10
        with open(p, "wb") as f:
            f.write(bytes(bad))
        with pytest.raises(RuntimeError, match=f"byte offset {spans[k][0]}:"):
            hostlib.bgzf_text(p, 1 << 20)


def test_windowed_reader_equals_the_reference_reader(tmp_path):
    import refh

    if not refh.available():
        pytest.skip("oracle/_ref/libmm_ref.so not built")
    R, H = refh.lib(), hostlib.lib()
    R.refh_read_file_digest.argtypes = [C.c_char_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    rng = np.random.default_rng(8)
    for v, text in enumerate([_fasta(rng, 80, [0, 61, 3000]), _fasta(rng, 20, [900], crlf=True, blank=True, final_newline=False)]):
        p = B.write_bgzf(tmp_path / f"v{v}.fa.gz", text, block=4000)
        want = [C.c_uint64() for _ in range(3)]
        assert R.refh_read_file_digest(p.encode(), *[C.byref(x) for x in want]) == 0
        got = [C.c_uint64() for _ in range(3)]
        assert H.skch_bgzf_read_digest(p.encode(), 5000, 2, *[C.byref(x) for x in got]) == 0
        assert [x.value for x in got] == [x.value for x in want]
