"""Writes tests/golden/align_band/edlib_digests.json: for every case of tests/test_gpu_align_band.py, the unmodified
edlib's result as [ed, sha256 of (ed, start, end, ops), sha256 of the standard CIGAR], keyed by
align_band_data.key(query, target, k, mode). The CLI case's regions come from the reference mapper's PAF (the same
mappings mashmap-b200 prints). Needs oracle/_ref (libedlib_nw_ref.so, libedlib_ref.so, mashmap_ref); no GPU.
Usage: python tests/golden/make_align_band_golden.py"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import align_band_data as AB  # noqa: E402
import align_data as AD  # noqa: E402
import align_nw_data as AN  # noqa: E402
from mashmap_b200 import capi  # noqa: E402


def main():
    assert AB.edlib_available(), "oracle/_ref is not built"
    out = {}

    def add(q, t, k, mode):
        out[AB.key(q, t, k, mode)] = e = AB.golden_entry(q, t, k, mode)
        return e

    NW, HW = capi.MM_ALIGN_NW, capi.MM_ALIGN_HW
    for name, q, t in AB.nw_pairs():
        ed = add(q, t, -1, NW)[0]
        if len(t) <= 2 * AB.L:
            for k in AB.k_variants(q, t, ed):
                add(q, t, k, NW)
        print(name, ed, flush=True)
    for name, q, t in AB.hw_pairs():
        for k in (-1, len(q)):
            print(name, add(q, t, k, HW)[0], flush=True)
    for name, q, t in AB.quirk_pairs():
        print(name, add(q, t, -1, NW)[0], flush=True)
    d = tempfile.mkdtemp()
    try:
        ref, qry = AB.write_asm(d)
        refs, queries = AN.read_fasta(ref), AN.read_fasta(qry)
        for mode, opts in sorted(AB.ASM_MODES.items()):
            paf = os.path.join(d, mode + ".paf")
            subprocess.run([AD.MAP_REF_BIN, "-r", ref, "-q", qry, "-o", paf, "-t", "8"] + AB.ASM_OPTS + opts,
                           check=True, capture_output=True, cwd=d)
            for q, t in AB.paf_regions(open(paf).read(), queries, refs):
                print(mode, len(q), len(t), add(q, t, -1, NW)[0], flush=True)
    finally:
        shutil.rmtree(d)
    os.makedirs(os.path.dirname(AB.GOLDEN), exist_ok=True)
    with open(AB.GOLDEN, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
