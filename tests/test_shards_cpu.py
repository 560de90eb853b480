"""--indexShards on the CPU: the shard plan, the refusals of the command line, and the frequent seeds of the whole
reference computed from per-shard key counts (the host step between the two device passes)."""
import os
import subprocess

import numpy as np
import pytest

import shard_data as S
from mashmap_b200 import hostlib, synth


def check_plan(first, lens, groups, by_group, n):
    C = len(lens)
    assert first[0] == 0 and first[-1] == C and len(first) == n + 1
    assert all(first[i] < first[i + 1] for i in range(n))  # contiguous, non-empty, ascending
    if by_group:
        for c in first[1:-1]:
            assert groups[c] != groups[c - 1], "a -Y prefix group spans two shards"
    return [int(np.sum(lens[first[i] : first[i + 1]])) for i in range(n)]


@pytest.mark.parametrize("seed", range(6))
def test_plan_is_contiguous_and_balanced(seed):
    rng = np.random.default_rng(seed)
    C = int(rng.integers(2, 40))
    lens = rng.integers(1_000, 1_000_000, size=C).astype(np.uint64)
    groups = np.zeros(C, dtype=np.int32)
    for n in range(1, C + 1):
        first = hostlib.plan_shards(lens, groups, False, n)
        bases = check_plan(first, lens, groups, False, n)
        # every cut is the contig boundary nearest its share of the bases, or as near as the cuts before it allow
        assert max(bases) <= int(lens.sum()) / n + 2 * int(lens.max())


@pytest.mark.parametrize("seed", range(6))
def test_plan_never_splits_a_prefix_group(seed):
    rng = np.random.default_rng(100 + seed)
    C = int(rng.integers(3, 30))
    lens = rng.integers(1_000, 500_000, size=C).astype(np.uint64)
    groups = np.cumsum(rng.random(C) < 0.4).astype(np.int32)  # runs of consecutive contigs
    runs = 1 + int(np.sum(groups[1:] != groups[:-1]))
    for n in range(1, runs + 1):
        check_plan(hostlib.plan_shards(lens, groups, True, n), lens, groups, True, n)
    with pytest.raises(ValueError, match=f"at most {runs} shards"):
        hostlib.plan_shards(lens, groups, True, runs + 1)


def test_plan_refuses_more_shards_than_contigs():
    lens = np.array([10, 20, 30], dtype=np.uint64)
    with pytest.raises(ValueError, match="at most 3 shards"):
        hostlib.plan_shards(lens, np.zeros(3, np.int32), False, 4)
    with pytest.raises(ValueError, match="at least one shard"):
        hostlib.plan_shards(lens, np.zeros(3, np.int32), False, 0)


@pytest.fixture(scope="module")
def small_set(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("shards"))
    genome = synth.random_genome(3, 20_000, seed=3)
    ref = os.path.join(d, "ref.fa")
    synth.write_fasta(ref, ["a#1", "a#2", "b#1"], genome)
    return d, ref


@pytest.mark.parametrize("extra,message", [
    (["--indexShards", "0"], "--indexShards needs a whole number of shards >= 1"),
    (["--indexShards", "two"], "--indexShards needs a whole number of shards >= 1"),
    (["--indexShards", "2", "--hostIndex"], "cannot be combined with --hostIndex, --saveIndex or --loadIndex"),
    (["--indexShards", "2", "--saveIndex", "PREFIX"], "cannot be combined with --hostIndex, --saveIndex or --loadIndex"),
    (["--indexShards", "2", "--loadIndex", "PREFIX"], "cannot be combined with --hostIndex, --saveIndex or --loadIndex"),
    (["--indexShards", "2", "--devices", "0-2"], "every device must hold a shard"),
    (["--indexShards", "4"], "at most 3 shards (2 possible cut points between contigs)"),
    (["--indexShards", "3", "-Y", "#"], "at most 2 shards (1 possible cut points between runs of contigs in different -Y prefix groups)"),
])
def test_cli_refuses_before_indexing(small_set, extra, message):
    d, ref = small_set
    out = os.path.join(d, "out.paf")
    p = subprocess.run([hostlib.CLI_PATH, "-r", ref, "-q", ref, "-s", "2000", "-o", out] + [x.replace("PREFIX", os.path.join(d, "ix")) for x in extra],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 1, p.stderr[-2000:]
    assert message in p.stderr, p.stderr[-2000:]
    assert "minmer windows picked" not in p.stderr


@pytest.mark.parametrize("which", ["panel", "repeat", "global_repeat"])
@pytest.mark.parametrize("pct", [1.0, 5.0, None])
def test_global_frequent_seeds_equal_the_whole_reference(tmp_path, which, pct):
    """per-shard key counts of random shardings, merged on the host: the same threshold and frequent set as the host
    builder over the whole reference (None: a threshold chosen so that per-shard thresholds would differ)"""
    import datasets

    if which == "global_repeat":
        genome = S.global_repeat_genome()[1]
    elif which == "panel":
        genome = datasets.make_panel_set(str(tmp_path))["genome"]
    else:
        genome = datasets.make_repeat_set(str(tmp_path))["genome"]
    if pct is None:
        pct = S.pick_pct(genome, [0, len(genome) // 2, len(genome)])
    t_whole, f_whole, keys_whole, _ = S.host_frequent(genome, pct)
    rng = np.random.default_rng(len(genome))
    for trial in range(3):
        n = int(rng.integers(2, len(genome) + 1))
        cuts = np.sort(rng.choice(np.arange(1, len(genome)), size=n - 1, replace=False)).tolist()
        first = [0] + cuts + [len(genome)]
        ks, cs = [], []
        for i in range(n):
            _, _, keys, cnt = S.host_frequent(genome[first[i] : first[i + 1]], pct)
            ks.append(keys)
            cs.append(cnt)
        t, uniq, freq = hostlib.global_frequent_seeds(ks, cs, pct)
        assert t == t_whole
        assert uniq == len(keys_whole)
        assert set(freq.tolist()) == f_whole
        assert list(freq) == sorted(freq)
