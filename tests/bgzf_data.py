"""BGZF (bgzip) files written with Python's zlib, and a corpus of raw DEFLATE blocks, for the BGZF reader's tests.

A BGZF member is a gzip member whose header carries FEXTRA with a 'BC' subfield of length 2 holding BSIZE (the member's
size minus 1); its data is one raw DEFLATE stream of at most 64 KiB of text, its trailer the CRC-32 and ISIZE. A file
ends with the 28-byte empty member (the EOF marker)."""
from __future__ import annotations

import struct
import zlib

import numpy as np

BLOCK = 65280  # bgzip's text per member: BSIZE stays below 64 KiB even for text that does not compress
EOF_MARKER = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def deflate_raw(text, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    co = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    return co.compress(text) + co.flush()


def member(text, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    data = deflate_raw(text, level, strategy)
    bsize = 18 + len(data) + 8 - 1
    assert bsize < 65536
    head = b"\x1f\x8b\x08\x04" + b"\x00" * 4 + b"\x00\xff" + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, bsize)
    return head + data + struct.pack("<II", zlib.crc32(text), len(text))


def bgzf(text, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, block=BLOCK, eof=True):
    out = [member(text[o : o + block], level, strategy) for o in range(0, len(text), block)]
    return b"".join(out) + (EOF_MARKER if eof else b"")


def write_bgzf(path, text, **kw):
    with open(path, "wb") as f:
        f.write(bgzf(text, **kw))
    return str(path)


def member_spans(blob):
    """(start, end) of each BGZF member of blob (its BSIZE fields)"""
    spans, p = [], 0
    while p + 18 <= len(blob) and blob[p : p + 2] == b"\x1f\x8b":
        bsize = struct.unpack_from("<H", blob, p + 16)[0]
        spans.append((p, p + bsize + 1))
        p += bsize + 1
    return spans


def dna(rng, n):
    return np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, n)].tobytes()


LEVELS = (0, 1, 6, 9)
STRATEGIES = {"fixed": zlib.Z_FIXED, "huffman": zlib.Z_HUFFMAN_ONLY, "rle": zlib.Z_RLE, "filtered": zlib.Z_FILTERED}


def corpus(seed=5, scale=1):
    """[(name, raw DEFLATE bytes, text)]: levels 0/1/6/9 and the four strategies over DNA text, FASTA text, random
    bytes, long runs (distance-1 matches), full 64 KiB blocks and empty ones; `scale` repeats the set with new text"""
    rng = np.random.default_rng(seed)
    out = []
    for rep in range(scale):
        texts = {
            "empty": b"",
            "one": b"A",
            "dna_full": dna(rng, BLOCK),
            "dna_65536": dna(rng, 65536),
            "dna_short": dna(rng, int(rng.integers(1, 5000))),
            "fasta": b"".join(b">r%d desc\n" % i + b"\n".join(dna(rng, 60) for _ in range(5)) + b"\n" for i in range(150))[:BLOCK],
            "random": rng.integers(0, 256, BLOCK, dtype=np.uint8).tobytes(),
            "runs": b"".join(bytes([int(rng.integers(65, 70))]) * int(rng.integers(1, 3000)) for _ in range(60))[:BLOCK],
            "repeat": (dna(rng, 37) * 2000)[:BLOCK],
        }
        for tname, text in texts.items():
            for level in LEVELS:
                out.append((f"{tname}_l{level}_{rep}", deflate_raw(text, level), text))
            for sname, strat in STRATEGIES.items():
                out.append((f"{tname}_{sname}_{rep}", deflate_raw(text, 6, strat), text))
    return out
