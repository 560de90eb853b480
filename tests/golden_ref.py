"""What the unmodified reference computed for the test data sets, stored as digests under tests/golden/ so that the tests
which compare the product with the reference still compare with it where the reference is not built (oracle/_ref needs
the reference's sources). tests/golden/make_reference_golden.py writes the file from the reference itself; with the
reference built, the tests compare with it directly and also check that the stored digests still agree with it.

A digest is the first 16 hex digits of the SHA-256 of the compared fields as int64, in the order the tests compare them."""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, "golden", "reference_digests.json")

SKETCH_FIELDS = ("hash", "wpos", "wpos_end", "strand")
L1_FIELDS = ("seqId", "rangeStartPos", "rangeEndPos", "intersectionSize")
L2_FIELDS = ("seqId", "meanOptimalPos", "optimalStart", "optimalEnd", "sharedSketchSize", "strand")

_store = None


def digest(*parts):
    h = hashlib.sha256()
    for p in parts:
        a = np.ascontiguousarray(np.asarray(p).astype(np.int64).reshape(-1))
        h.update(np.int64(a.size).tobytes())
        h.update(a.tobytes())
    return h.hexdigest()[:16]


def sketch_digest(sk, n=None):
    sk = sk if n is None else sk[:n]
    return digest(len(sk), *[sk[f] for f in SKETCH_FIELDS])


def fragment_digest(sketch, sketch_size, n_points, l1, l2_per_candidate):
    """one query fragment through K1 -> K2 -> K3: sketch after the frequent-seed drop, its size, the number of interval
    points, the L1 candidates and, candidate by candidate, the L2 loci"""
    parts = [sketch_size, n_points, len(l1)] + [sketch[f] for f in SKETCH_FIELDS] + [l1[f] for f in L1_FIELDS]
    for rows in l2_per_candidate:
        parts += [len(rows)] + [rows[f] for f in L2_FIELDS]
    return digest(*parts)


def reference_fragment_digest(o):
    """fragment_digest of refh.RefSession.map_fragment's output"""
    l2 = [o["l2"][o["l2_cand"] == ci] for ci in range(len(o["l1"]))]
    return fragment_digest(o["sketch"], len(o["sketch"]), o["n_points"], o["l1"], l2)


def index_digests(mi, keys, offs, pts, fr, freq_threshold):
    """minmerIndex as a multiset per (seqId, wpos, wpos_end) group (the order inside a group of ties is std::sort's), the
    lookup table exactly"""
    order = np.lexsort((mi["strand"], mi["hash"], mi["wpos_end"], mi["wpos"], mi["seqId"]))
    m = mi[order]
    return {"n_minmers": int(len(mi)), "minmers": digest(*[m[f] for f in ("seqId", "wpos", "wpos_end", "hash", "strand")]),
            "keys": digest(keys), "offs": digest(offs), "points": digest(*[pts[f] for f in ("pos", "seqId", "side", "hash")]),
            "is_freq": digest(np.asarray(fr).astype(np.int64)), "freq_threshold": int(freq_threshold)}


def key_of(args, d=None):
    """a command line with the data set's temporary paths replaced by their file names"""
    paths = {} if d is None else {d["ref"]: os.path.basename(d["ref"]), d["qry"]: os.path.basename(d["qry"])}
    return " ".join(paths.get(a, a) for a in args)


def load():
    global _store
    if _store is None:
        _store = json.load(open(PATH)) if os.path.exists(PATH) else {}
    return _store


def get(section, key):
    v = load().get(section, {}).get(key)
    assert v is not None, f"no stored reference result for {section} / {key}: run tests/golden/make_reference_golden.py"
    return v


def check_stored(section, key, value):
    """with the reference built: the stored digests must still be what the reference computes"""
    stored = load().get(section, {}).get(key)
    if stored is not None:
        assert stored == value, f"tests/golden/reference_digests.json is stale for {section} / {key}"


class ProductSession:
    """Stands in for refh.RefSession where the reference is not built: the same command line through the product's own
    host program (parameters, skch::Sketch from the FASTA files, cutoff and minimum-hits tables). Whatever the tests take
    from it is checked against the reference's stored digests (parameters, index, tables) before it is used."""

    def __init__(self, args):
        from mashmap_b200 import hostlib

        import refh

        self._hl = hostlib
        self.key = None
        self.hi = hostlib.HostIndex.from_cli(args)
        self.p = self.hi.params_into(refh.OrcParams())
        self._arrays = None

    def close(self):
        pass

    def _a(self):
        if self._arrays is None:
            self._arrays = self.hi.arrays()
        return self._arrays

    def index(self):
        return self._a()[0]

    def lookup(self):
        return self._a()[1:]

    def freq_threshold(self):
        return self.hi.freq_threshold

    def cutoffs(self):
        p = self.p
        return self._hl.sketch_cutoffs(p.sketchSize, p.kmerSize, p.ANIDiff, p.ANIDiffConf, bool(p.stage1_topANI_filter))

    def min_hits_table(self):
        return self._hl.min_hits_table(self.p.sketchSize, self.p.kmerSize, self.p.percentageIdentity)


def session_digests(R):
    """what a session hands the device: parameters, index, tables"""
    p = R.p
    mi = R.index()
    keys, offs, pts, fr = R.lookup()
    return {"params": [int(p.kmerSize), int(p.segLength), int(p.sketchSize), float(p.percentageIdentity), int(p.stage1_topANI_filter)],
            "index": index_digests(mi, keys, offs, pts, fr, R.freq_threshold()),
            "tables": digest(R.cutoffs(), R.min_hits_table())}
