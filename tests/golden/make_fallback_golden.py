"""Writes the reference's results for the tandem repeat sets of tests/test_gpu_fallbacks.py (make_repeat_set with 16, 17
and 24 tandem copies, --noHgFilter) from the UNMODIFIED reference (oracle/_ref, built by `make -C oracle ref` where the
reference's sources are), next to the entries of the other golden scripts:
  tests/golden/reference_digests.json  the digests of what a session hands the device and of the reference's stages per
                                       split fragment (tests/golden_ref.py)
  tests/golden/nosplit_digests.json    the digests of the reference's stages per whole query (what --noSplit maps)
Run: python tests/golden/make_fallback_golden.py"""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import golden_ref  # noqa: E402
import refh  # noqa: E402
import fallback_data as FD  # noqa: E402
import nosplit_data as ND  # noqa: E402
from mashmap_b200 import synth  # noqa: E402

assert refh.available(), "oracle/_ref/libmm_ref.so is not built"
wd = tempfile.mkdtemp(prefix="mm_fallback_golden_")
store = golden_ref.load()
whole_store = ND.load()
for n in FD.TANDEM_COPIES:
    d = FD.tandem_set(wd, n)
    args = FD.tandem_args(d)
    key = golden_ref.key_of(args, d)
    R = refh.RefSession(args)
    store["sessions"][key] = golden_ref.session_digests(R)
    lens = [len(r) for r in d["reads"]]
    ridx, start, length = synth.split_segments(lens, R.p.segLength, R.p.kmerSize)
    store["fragments"][key] = [golden_ref.reference_fragment_digest(
        R.map_fragment(d["rnames"][ridx[i]], d["reads"][ridx[i]][start[i] : start[i] + length[i]], full_len=lens[ridx[i]],
                       seq_counter=int(ridx[i]))) for i in range(len(ridx))]
    wi, wl = ND.whole_reads(d, R.p.kmerSize)
    outs = [R.map_fragment(d["rnames"][i], d["reads"][i], full_len=int(n), seq_counter=int(i)) for i, n in zip(wi, wl)]
    whole_store["fragments"][key] = [golden_ref.reference_fragment_digest(o) for o in outs]
    most = max((int(np.bincount(o["l2_cand"]).max()) for o in outs if len(o["l2_cand"])), default=0)
    print(f"{key}: s = {R.p.sketchSize}, {len(ridx)} fragments, {len(wi)} whole queries, most loci of one whole-query "
          f"candidate {most}", flush=True)
    R.close()
json.dump(store, open(golden_ref.PATH, "w"), separators=(",", ":"), sort_keys=True)
print("wrote", golden_ref.PATH, os.path.getsize(golden_ref.PATH), "bytes")
json.dump(whole_store, open(ND.PATH, "w"), separators=(",", ":"), sort_keys=True)
print("wrote", ND.PATH, os.path.getsize(ND.PATH), "bytes")
