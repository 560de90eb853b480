"""Data for the contig-sharded index (--indexShards) tests: a reference whose frequent seeds differ between a per-shard and
a whole-reference frequency threshold, and helpers shared by the CPU and GPU files."""
import os

import numpy as np

from mashmap_b200 import synth

K, SEG, SKETCH = 19, 1000, 60
N_CONTIGS, CONTIG_LEN = 4, 60_000
ELEMENT_LEN = 1500


def global_repeat_genome(seed=71):
    """Element A: 3 exact copies in every contig (12 in all). Element B: 7 exact copies in contig 0 only. Over the whole
    reference A's hashes are the most frequent (24 interval points against B's 14); over contigs 0-1 alone B's are (14
    against 12): a threshold taken per shard flags B there and leaves A in, one taken over the whole reference flags A."""
    rng = np.random.default_rng(seed)
    a = synth.random_sequence(ELEMENT_LEN, rng)
    b = synth.random_sequence(ELEMENT_LEN, rng)
    contigs = []
    for c in range(N_CONTIGS):
        s = synth.random_sequence(CONTIG_LEN, rng)
        n_b = 7 if c == 0 else 0
        slots = np.sort(rng.choice(np.arange(1, CONTIG_LEN // (2 * ELEMENT_LEN) - 1), size=3 + n_b, replace=False))
        kinds = ["A"] * 3 + ["B"] * n_b
        rng.shuffle(kinds)
        for at, kind in zip(slots, kinds):
            s[at * 2 * ELEMENT_LEN : at * 2 * ELEMENT_LEN + ELEMENT_LEN] = a if kind == "A" else b
        contigs.append(s)
    names = [f"ctg{c}" for c in range(N_CONTIGS)]
    return names, contigs


def offsets(seqs):
    o = np.zeros(len(seqs) + 1, dtype=np.uint64)
    o[1:] = np.cumsum([len(s) for s in seqs])
    return o


def key_counts(offs):
    return (offs[1:] - offs[:-1]).astype(np.uint32)


def host_frequent(seqs, pct):
    """(threshold, frequent hashes) of the host builder over these contigs"""
    from mashmap_b200 import hostlib

    h = hostlib.HostIndex.build(np.concatenate(seqs), offsets(seqs), K, SEG, SKETCH, kmer_pct_threshold=pct)
    _, keys, offs, _, fr = h.arrays()
    t = h.freq_threshold
    h.close()
    return t, set(keys[fr.astype(bool)].tolist()), keys, key_counts(offs)


def pick_pct(genome, first):
    """a --kmerThreshold whose frequent seeds over the whole reference differ from those that thresholds taken over each
    shard of the plan `first` alone would give (the case a per-shard build gets wrong)"""
    _, _, _, cnt = host_frequent(genome, 0.001)
    for c in sorted(set(cnt.tolist()), reverse=True)[:12]:
        pct = 100.0 * (int((cnt >= c).sum()) + 0.5) / len(cnt)
        _, whole, _, _ = host_frequent(genome, pct)
        for i in range(len(first) - 1):
            _, own, keys, _ = host_frequent(genome[first[i] : first[i + 1]], pct)
            if own != whole & set(keys.tolist()):
                return pct
    raise AssertionError("no threshold separates the per-shard and the global frequent seeds")


def write_set(workdir, tag="gfreq"):
    names, contigs = global_repeat_genome()
    rng = np.random.default_rng(72)
    reads, rnames = [], []
    for i in range(24):  # 4 kb reads across every contig, many over a copy of A or B
        c = i % N_CONTIGS
        at = int(rng.integers(0, CONTIG_LEN - 4000))
        reads.append(synth.mutate(contigs[c][at : at + 4000], 0.01, rng)[:4000])
        rnames.append(f"r{i}_{c}_{at}")
    ref = os.path.join(workdir, f"{tag}_ref.fa")
    qry = os.path.join(workdir, f"{tag}_reads.fa")
    synth.write_fasta(ref, names, contigs)
    synth.write_fasta(qry, rnames, reads)
    return dict(ref=ref, qry=qry, genome=contigs, names=names, reads=reads, rnames=rnames)
