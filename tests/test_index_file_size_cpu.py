"""--loadIndex on the host path (--hostIndex, as HostIndex.from_cli builds it) checks PREFIX.index's size against its
header's record count before it allocates anything: a file too short for the records its header counts stops with exit
status 1 and a message naming the file and its size. Bytes after the records are ignored, as in the reference, and so
are the records' _pad bytes. CPU only."""
import os
import subprocess
import sys

import numpy as np
import pytest

import datasets
from mashmap_b200 import capi, hostlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = ("import sys; from mashmap_b200 import hostlib; h = hostlib.HostIndex.from_cli(sys.argv[1:]); "
         "print(h.n_minmers, h.n_keys, h.n_points, h.freq_threshold)")


def load_in_child(args):
    """HostIndex.from_cli in a process of its own: a refused file ends that process"""
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-s", "-c", CHILD] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                          env=env, cwd=ROOT)


@pytest.fixture(scope="module")
def saved(workdir):
    d = datasets.make_random_set(workdir, tag="ifs", n_reads=2)
    base = ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "-t", "3"]
    prefix = os.path.join(workdir, "ifs_saved")
    h = hostlib.HostIndex.from_cli(base + ["--saveIndex", prefix])
    want = f"{h.n_minmers} {h.n_keys} {h.n_points} {h.freq_threshold}"
    h.close()
    with open(prefix + ".index", "rb") as f:
        raw = f.read()
    assert int(np.frombuffer(raw[:8], dtype=np.uint64)[0]) * 24 + 8 == len(raw) > 8
    return base, raw, want


def write_variant(workdir, saved, tag, blob):
    prefix = os.path.join(workdir, "ifs_" + tag)
    with open(prefix + ".index", "wb") as f:
        f.write(blob)
    return prefix


def test_a_well_formed_file_loads(workdir, saved):
    base, raw, want = saved
    p = load_in_child(base + ["--loadIndex", write_variant(workdir, saved, "same", raw)])
    assert p.returncode == 0, p.stderr[-1000:]
    assert p.stdout.split("\n")[0] == want


def test_trailing_bytes_and_pad_bytes_are_ignored(workdir, saved):
    base, raw, want = saved
    mi = np.frombuffer(raw[8:], dtype=capi.minmer_dtype).copy()
    mi["_pad"] = np.arange(len(mi)) % 30000 + 1
    blob = raw[:8] + mi.tobytes() + b"trailing bytes after the records"
    p = load_in_child(base + ["--loadIndex", write_variant(workdir, saved, "tail", blob)])
    assert p.returncode == 0, p.stderr[-1000:]
    assert p.stdout.split("\n")[0] == want


@pytest.mark.parametrize("case", ["truncated", "count_too_large", "no_header"])
def test_a_file_too_short_for_its_header_is_refused(workdir, saved, case):
    base, raw, _ = saved
    n = int(np.frombuffer(raw[:8], dtype=np.uint64)[0])
    blob = {"truncated": raw[:-1],
            "count_too_large": np.array([1 << 61], dtype=np.uint64).tobytes() + raw[8:],
            "no_header": raw[:5]}[case]
    prefix = write_variant(workdir, saved, case, blob)
    p = load_in_child(base + ["--loadIndex", prefix])
    assert p.returncode == 1, (p.returncode, p.stderr[-1000:])
    assert prefix + ".index" in p.stderr and f"holds {len(blob)} bytes" in p.stderr, p.stderr[-1000:]
    if case != "no_header":
        assert str(n if case == "truncated" else 1 << 61) + " records" in p.stderr
