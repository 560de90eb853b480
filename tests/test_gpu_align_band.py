"""Long alignments on the device: NW sub-problems with max(Q, T) >= MM_ALIGN_BAND_MIN_LEN run banded, one CTA per
sweep (DESIGN.md section 10). Results are checked against the unmodified edlib (oracle/_ref) where it is built, and
against the digests of its results in tests/golden/align_band/ otherwise (align_band_data.want)."""
import os
import re
import subprocess

import numpy as np
import pytest

import align_band_data as AB
import align_nw_data as AN
import align_data as AD
from conftest import have_gpu
from mashmap_b200 import capi

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_gpu(), reason="no GPU")]

MAP_BIN = os.path.join(AD.ROOT, "mashmap_b200", "mashmap-b200")


def _jobs(cases):
    """cases: (query, target, k, mode)"""
    qb = np.concatenate([c[0] for c in cases])
    tb = np.concatenate([c[1] for c in cases])
    jobs = np.zeros(len(cases), dtype=capi.align_job_dtype)
    jobs["q_len"] = [len(c[0]) for c in cases]
    jobs["t_len"] = [len(c[1]) for c in cases]
    jobs["q_offset"][1:] = np.cumsum(jobs["q_len"].astype(np.int64))[:-1]
    jobs["t_offset"][1:] = np.cumsum(jobs["t_len"].astype(np.int64))[:-1]
    jobs["k"] = [c[2] for c in cases]
    jobs["mode"] = [c[3] for c in cases]
    return qb, tb, jobs


def _results(ctx, cases):
    res, ops = ctx.align(*_jobs(cases))
    out = []
    for r in res:
        o = int(r["ops_offset"])
        out.append((int(r["ed"]), int(r["start"]), int(r["end"]), ops[o : o + int(r["alignment_length"])].copy()))
    return out


def _check(cases, got, names):
    for c, g, name in zip(cases, got, names):
        ed, d, _ = AB.want(*c)
        assert g[0] == ed, (name, len(c[0]), len(c[1]), c[2], g[0], ed)
        assert AB.digest(*g) == d, (name, len(c[0]), len(c[1]), c[2])
        if g[0] >= 0 and c[3] == capi.MM_ALIGN_NW:
            assert AN.cigar_lengths(AD.cigar(g[3])) == (len(c[0]), len(c[1])), name


def test_nw_pairs_straddling_the_rule_equal_edlib():
    """NW pairs of lengths L - 1 (warp path) to 1 Mbp at 0-15 %, k = -1, then k = ed, ed - 1 and |Q - T| - 1 for the
    pairs up to 2L; one batch of all of them"""
    pairs = AB.nw_pairs()
    ctx = capi.AlignContext(0)
    cases = [(q, t, -1, capi.MM_ALIGN_NW) for _, q, t in pairs]
    names = [n for n, _, _ in pairs]
    got = _results(ctx, cases)
    _check(cases, got, names)
    assert any(len(q) >= AB.L for _, q, _ in pairs) and any(max(len(q), len(t)) < AB.L for _, q, t in pairs)
    more, more_names = [], []
    for (name, q, t), g in zip(pairs, got):
        if len(t) <= 2 * AB.L:
            for k in AB.k_variants(q, t, g[0]):
                more.append((q, t, k, capi.MM_ALIGN_NW))
                more_names.append(f"{name}_k{k}")
    got2 = _results(ctx, more)
    _check(more, got2, more_names)
    assert sum(g[0] < 0 for g in got2) >= 10  # ed - 1 and below the length difference
    ctx.close()


def test_hw_jobs_with_long_hirschberg_nodes_equal_edlib():
    ctx = capi.AlignContext(0)
    pairs = AB.hw_pairs()
    cases = [(q, t, k, capi.MM_ALIGN_HW) for _, q, t in pairs for k in (-1, len(q))]
    got = _results(ctx, cases)
    _check(cases, got, [n for n, _, _ in pairs for _ in (0, 1)])
    assert all(g[0] > 0 for g in got)
    ms = ctx.stage_ms()
    assert ms[7] >= 3  # several Hirschberg levels
    ctx.close()


def test_long_and_short_jobs_mixed_and_in_waves_give_what_they_give_alone():
    rng = np.random.default_rng(31)
    long_pairs = AB.nw_pairs()[5:12] + AB.hw_pairs()[:1]
    cases = []
    for i, (_, q, t) in enumerate(long_pairs):
        cases.append((q, t, -1, capi.MM_ALIGN_HW if i == len(long_pairs) - 1 else capi.MM_ALIGN_NW))
    for i in range(300):
        q, t = AD.threshold_pair(rng) if i % 50 == 0 else AD.random_pair(rng)
        cases.append((q, t, -1 if i % 3 else len(q), capi.MM_ALIGN_NW if i % 2 else capi.MM_ALIGN_HW))
    order = rng.permutation(len(cases))
    mixed = [cases[i] for i in order]
    ctx = capi.AlignContext(0)
    alone = [_results(ctx, [c])[0] for c in cases[: len(long_pairs)]]
    alone += _results(ctx, cases[len(long_pairs) :])
    got = _results(ctx, mixed)
    small = capi.AlignContext(0, 1)  # the smallest scratch budget: every stage runs in waves
    got_small = _results(small, mixed)
    for j, i in enumerate(order):
        for g in (got[j], got_small[j]):
            assert g[:3] == alone[i][:3] and np.array_equal(g[3], alone[i][3]), (i, len(cases[i][0]))
    ctx.close()
    small.close()


def test_edlib_quirks_on_the_long_path():
    """a 3 Mbp pair at 0.5 % equals edlib; a 3.4 Mbp query against a 2-base target (a one-column Hirschberg node below
    the root) gives the exact distance and no path"""
    pairs = AB.quirk_pairs()
    cases = [(q, t, -1, capi.MM_ALIGN_NW) for _, q, t in pairs]
    ctx = capi.AlignContext(0)
    got = _results(ctx, cases)
    _check(cases, got, [n for n, _, _ in pairs])
    assert got[0][0] > 0 and len(got[0][3]) >= len(pairs[0][1])
    q, t = AB.one_column_pair()
    ed, start, end, ops = _results(ctx, [(q, t, -1, capi.MM_ALIGN_NW)])[0]
    # the target is the query's first two bases: the distance is |Q - T| (match both, insert the rest)
    assert (ed, start, end, len(ops)) == (len(q) - 2, 0, 1, 0)
    ctx.close()


# ---- the CLI on assembly-like contigs --------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def asm(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("align_band"))
    ref, qry = AB.write_asm(d)
    return dict(dir=d, ref=ref, qry=qry, refs=AN.read_fasta(ref), queries=AN.read_fasta(qry))


def _map(asm, opts):
    out = os.path.join(asm["dir"], "out.paf")
    p = subprocess.run([MAP_BIN, "-r", asm["ref"], "-q", asm["qry"], "-o", out] + AB.ASM_OPTS + opts,
                       capture_output=True, text=True, cwd=asm["dir"])
    assert p.returncode == 0, p.stderr[-3000:]
    return open(out).read(), p.stderr


@pytest.mark.parametrize("mode", sorted(AB.ASM_MODES))
def test_cli_aligns_assembly_scale_mappings(asm, mode):
    plain, _ = _map(asm, AB.ASM_MODES[mode])
    text, err = _map(asm, AB.ASM_MODES[mode] + ["--align", "--alignMaxLen", "5000000"])
    assert AN.strip_tags(text) == plain
    assert "; 0 mappings with a region longer than --alignMaxLen 5000000 " in err, err[-2000:]
    lens = [max(int(f[3]) - int(f[2]), int(f[8]) - int(f[7])) for f in (ln.split("\t") for ln in text.splitlines())]
    assert max(lens) > 1_000_000 and len(lens) >= 3
    if AB.edlib_available():
        tagged, untagged = AN.check_tags(text, asm["queries"], asm["refs"])
        assert tagged == len(lens) and untagged == 0
    else:
        for line, (q, t) in zip(text.splitlines(), AB.paf_regions(text, asm["queries"], asm["refs"])):
            nm, cg = re.search(r"\tNM:i:(\d+)\tcg:Z:([0-9MID]*)$", line).groups()
            assert AN.cigar_lengths(cg) == (len(q), len(t)), line[:200]
            ed, _, cd = AB.want(q, t, -1, capi.MM_ALIGN_NW)
            assert int(nm) == ed and AB.cigar_digest(cg) == cd, line[:200]
