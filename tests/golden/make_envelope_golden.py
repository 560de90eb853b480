"""Writes the reference's results for the envelope tests (tests/test_gpu_envelope.py, data in tests/envelope_data.py)
from the UNMODIFIED reference (oracle/_ref, built by `make -C oracle ref` where the reference's sources are):
  sessions, fragments  for every stage-parity row: the digests of what a session hands the device and of the reference's
                       stages per fragment (tests/golden_ref.py), added to tests/golden/reference_digests.json next to
                       the entries tests/golden/make_reference_golden.py writes
  envelope/*.paf       the reference CLI's output for every envelope_data.CLI_RUNS command line
Needs the product's CUDA library (for the largest sketch size mm_params_check accepts), no GPU.
Run: python tests/golden/make_envelope_golden.py"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import envelope_data as ED  # noqa: E402
import golden_ref  # noqa: E402
import refh  # noqa: E402
from mashmap_b200 import synth  # noqa: E402

assert refh.available(), "oracle/_ref/libmm_ref.so is not built"
wd = tempfile.mkdtemp(prefix="mm_envelope_golden_")
data = ED.datasets_by_name(wd)
store = golden_ref.load()
for row, which, opts, _ in ED.stage_runs():
    d = data(which)
    args = ["-r", d["ref"], "-q", d["qry"]] + opts
    key = golden_ref.key_of(args, d)
    R = refh.RefSession(args)
    store["sessions"][key] = golden_ref.session_digests(R)
    lens = [len(r) for r in d["reads"]]
    ridx, start, length = synth.split_segments(lens, R.p.segLength, R.p.kmerSize)
    store["fragments"][key] = [golden_ref.reference_fragment_digest(
        R.map_fragment(d["rnames"][ridx[i]], d["reads"][ridx[i]][start[i] : start[i] + length[i]], full_len=lens[ridx[i]],
                       seq_counter=int(ridx[i]))) for i in range(len(ridx))]
    print(f"{row}: {key}: s = {R.p.sketchSize}, {len(ridx)} fragments", flush=True)
    R.close()
json.dump(store, open(golden_ref.PATH, "w"), separators=(",", ":"), sort_keys=True)
print("wrote", golden_ref.PATH, os.path.getsize(golden_ref.PATH), "bytes")
os.makedirs(ED.PAF_DIR, exist_ok=True)
for which, opts in ED.CLI_RUNS:
    d = data(which)
    dst = os.path.join(ED.PAF_DIR, ED.cli_name(which, opts) + ".paf")
    subprocess.run([refh.REF_BIN, "-r", d["ref"], "-q", d["qry"], "-t", "8", "-o", dst] + opts, check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    print("wrote", dst, os.path.getsize(dst), "bytes", flush=True)
