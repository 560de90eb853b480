"""What a mapping context can run, answered before any device work (mm_params_check): every mapping kernel whose launch
size depends on (seg_length, sketch_size, kmer_size) -- K1, K2's general path, the general L2 kernel (its live set and its
shared memory), the L2 kernel of long fragments -- through the size functions their launchers use. CPU only."""
import os
import re
import subprocess

import pytest

import envelope_data as ED
from mashmap_b200 import capi, hostlib, synth

SEGS = [100, 101, 150, 500, 1000, 2000, 5000, 10000, 20000, 50000, 100000]
# every size up to 300 (tiny sketches, k_l1_warp's hit-list switch at 256 / 257), then a coarse sweep to 15,000 and each
# switch with its neighbours: the stream kernel's 11-bit counters (1000), the general L2 kernel's shared memory (~1964)
# and live set (1985, 2048), the reference's cut-off table step (2000), K2's general path (~11,900)
S_GRID = sorted(set(range(1, 301)) | set(range(300, 15001, 97))
                | {s + d for s in (1000, 1964, 1985, 2000, 2048, 11900, 15000) for d in range(-3, 4)})
REFUSED = re.compile(r"seg_length (\d+) / sketch_size (\d+) exceed the shared-memory budget of (.+?); (?:the largest sketch "
                     r"size accepted for seg_length (\d+) \(k = (\d+)\) is (\d+)|no sketch size is accepted)")


def check(k, seg, s):
    return capi.params_check(k, seg, s)


@pytest.mark.parametrize("k", list(range(8, 33)))
def test_acceptance_is_monotone_in_sketch_size_and_the_message_names_the_limit(k):
    """for every k-mer size and segment length: the accepted sketch sizes are 1..S_max (nothing larger is accepted once a
    size is refused), and every refusal names a kernel and S_max itself, which is accepted while S_max + 1 is not"""
    for seg in SEGS:
        refused_at = None
        for s in S_GRID:
            rc, msg = check(k, seg, s)
            if rc == capi.MM_OK:
                assert refused_at is None, (k, seg, s, "accepted after", refused_at)
                continue
            assert rc == capi.MM_EINVAL
            m = REFUSED.match(msg)
            assert m, msg
            assert (int(m.group(1)), int(m.group(2))) == (seg, s)
            if refused_at is None:
                refused_at = s
                if m.group(6) is None:
                    assert check(k, seg, 1)[0] != capi.MM_OK
                    s_max = 0
                else:
                    s_max = int(m.group(6))
                    assert (int(m.group(4)), int(m.group(5))) == (seg, k)
                    assert check(k, seg, s_max)[0] == capi.MM_OK and check(k, seg, s_max + 1)[0] != capi.MM_OK
                assert s_max < s
            elif m.group(6) is not None:
                assert int(m.group(6)) == s_max
        # the general L2 kernel bounds every segment length: nothing above its limit is ever accepted
        assert refused_at is not None and refused_at <= 1965


def test_general_l2_limit():
    """k_l2 holds four warps of (S + 2) * 21 bytes of query sketch, a live set of roundup32(S + 64) * 8 bytes and a
    384-byte staging area in 227 KB: S = 1964 is the last size that fits, the same at every segment length K1 fits"""
    for seg in (1000, 5000, 20000):
        assert ED.largest_sketch_size(seg) == 1964
        rc, msg = check(19, seg, 1965)
        assert rc == capi.MM_EINVAL and "general L2 kernel" in msg and msg.endswith("is 1964"), msg


@pytest.fixture(scope="module")
def env(workdir):
    return ED.datasets_by_name(workdir)


def parsed_params(args):
    """(k, seg_length, sketch_size) the product's option parser derives for a command line, as the reference does"""
    from refh import OrcParams

    p = hostlib.HostIndex.params_from_cli(args).params_into(OrcParams())
    return int(p.kmerSize), int(p.segLength), int(p.sketchSize)


def test_every_envelope_row_is_accepted(env):
    """every stage-parity and CLI row of the GPU envelope tests is inside the envelope, at the sketch size the option
    parser picks; the reference's own rule gives s = 998 and 1598 there"""
    rows = [(w, o) for _, w, o, _ in ED.stage_runs()] + ED.CLI_RUNS
    for which, opts in rows:
        d = env(which)
        k, seg, s = parsed_params(["-r", d["ref"], "-q", d["qry"]] + opts)
        assert check(k, seg, s) == (capi.MM_OK, ""), (which, opts, k, seg, s)
    d = env("reads")
    assert parsed_params(["-r", d["ref"], "-q", d["qry"], "-s", "10000", "--dense", "--pi", "80"])[2] == 998
    assert parsed_params(["-r", d["ref"], "-q", d["qry"], "-s", "20000", "--dense", "--pi", "85"])[2] == 1598


@pytest.mark.parametrize("opts,s", [(["-s", "5000", "-J", "2000"], 2000), (["-s", "20000", "--dense", "--pi", "80"], 1998),
                                    (["-s", "30000", "--dense", "--pi", "85"], 2398)])
def test_sketch_sizes_past_the_general_l2_kernel_are_refused(env, opts, s):
    d = env("reads")
    k, seg, got = parsed_params(["-r", d["ref"], "-q", d["qry"]] + opts)
    assert got == s
    rc, msg = check(k, seg, s)
    assert rc == capi.MM_EINVAL and "general L2 kernel (K3)" in msg and msg.endswith("is 1964"), msg


def test_cli_refuses_before_reading_the_reference(workdir):
    """`-s 5000 -J 2000`: the CLI stops with the parameter check's message and exit status 1 before it reads or indexes
    the reference (the check runs first and needs no device, so this holds on a machine without a GPU too)"""
    import numpy as np

    rng = np.random.default_rng(3)
    fa = os.path.join(workdir, "tiny_limits.fa")
    synth.write_fasta(fa, ["c0"], [synth.random_sequence(20_000, rng)])
    out = os.path.join(workdir, "tiny_limits.paf")
    p = subprocess.run([hostlib.CLI_PATH, "-r", fa, "-q", fa, "-s", "5000", "-J", "2000", "-t", "2", "-o", out],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 1, p.stderr[-2000:]
    assert "[mashmap-b200] ERROR: seg_length 5000 / sketch_size 2000 exceed the shared-memory budget of the general L2 " \
           "kernel (K3); the largest sketch size accepted for seg_length 5000 (k = 19) is 1964" in p.stderr, p.stderr[-2000:]
    assert "minmer windows picked from reference" not in p.stderr + p.stdout  # the reference was not indexed
    assert not os.path.exists(out) or os.path.getsize(out) == 0


def test_oracle_cut_off_table_is_exact_at_large_sketch_sizes():
    """The hypergeometric cut-off table from s = 900 on: the GSL stand-in the oracle and the reference are built with
    (oracle/gsl_shim) equals the product's table, and at the entries where a subnormal start term used to move the
    stand-in's sum, both equal the decision computed in exact rational arithmetic (computeMap.hpp:199-253, min_p the
    float 1 - 0.999)"""
    from fractions import Fraction
    from math import comb

    import numpy as np

    import oracle_py

    for ss in (900, 1000):
        O = oracle_py.Oracle(sketch_size=ss)
        try:
            assert np.array_equal(O.cutoffs(), hostlib.sketch_cutoffs(ss, 19, 0.0, 0.999, True)), ss
        finally:
            O.close()
    ss, min_p = 1000, Fraction(float(np.float32(1) - np.float32(0.999)))

    def pmf(t):
        return [Fraction(comb(ss, y) * comb(ss - t, t - y), comb(2 * ss - t, t)) for y in range(t + 1)]

    def above(cmax, ci):  # Pr(Y_ci >= Y_cmax) > min_p
        pm, pc = pmf(cmax), pmf(ci)
        tail, acc = [Fraction(1)], Fraction(0)
        for y in range(1, cmax + 1):
            acc += pc[y - 1] if y - 1 <= ci else 0
            tail.append(1 - acc)
        return sum(pm[y] * tail[y] for y in range(cmax + 1)) > min_p

    cut = hostlib.sketch_cutoffs(ss, 19, 0.0, 0.999, True)
    for cmax in (510, 565):
        ci = int(cut[cmax])
        assert above(cmax, ci) and not above(cmax, ci - 1), (cmax, ci)
