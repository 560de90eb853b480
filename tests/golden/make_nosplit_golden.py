"""Writes tests/golden/nosplit_digests.json and tests/golden/nosplit/*.paf from the UNMODIFIED reference (oracle/_ref, built
by `make -C oracle ref` where the reference's sources are), for the tests of queries mapped as one fragment longer than a
segment (tests/test_gpu_nosplit.py):
  sketch_long  digests (tests/golden_ref.py) of CommonFunc::sketchSequence over the fragments of nosplit_data.long_sequences
  fragments    per whole query of the STAGE_RUNS data sets: the digest of the reference's stages (mapSingleQueryFrag on
               the whole query: sketch, points, L1 candidates, L2 loci per candidate)
  *.paf        the reference CLI's output with --noSplit for every CLI_RUNS command line
No GPU needed. Run: python tests/golden/make_nosplit_golden.py"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import golden_ref  # noqa: E402
import nosplit_data as ND  # noqa: E402
import refh  # noqa: E402

assert refh.available(), "oracle/_ref/libmm_ref.so is not built"
wd = tempfile.mkdtemp(prefix="mm_nosplit_golden_")
sets = {}
make = ND.datasets_by_name(wd)


def data(name):
    if name not in sets:
        sets[name] = make[name]()
    return sets[name]


out = {"sketch_long": {}, "fragments": {}}
for k, s in ND.SKETCH_CASES:
    out["sketch_long"][f"k{k} s{s}"] = [golden_ref.sketch_digest(refh.sketch_sequence(q, k, s, seq_id=i))
                                        for i, q in enumerate(ND.long_sequences(k))]
for name, opts in ND.STAGE_RUNS:
    d = data(name)
    args = ["-r", d["ref"], "-q", d["qry"]] + opts
    R = refh.RefSession(args)
    ridx, lens = ND.whole_reads(d, R.p.kmerSize)
    out["fragments"][golden_ref.key_of(args, d)] = [golden_ref.reference_fragment_digest(
        R.map_fragment(d["rnames"][i], d["reads"][i], full_len=int(n), seq_counter=int(i))) for i, n in zip(ridx, lens)]
    R.close()
    print(name, opts, len(ridx), "queries", flush=True)
json.dump(out, open(ND.PATH, "w"), separators=(",", ":"), sort_keys=True)
print("wrote", ND.PATH, os.path.getsize(ND.PATH), "bytes")
os.makedirs(ND.PAF_DIR, exist_ok=True)
for name, opts in ND.CLI_RUNS:
    d = data(name)
    dst = os.path.join(ND.PAF_DIR, ND.cli_name(name, opts) + ".paf")
    subprocess.run([refh.REF_BIN, "-r", d["ref"], "-q", d["qry"], "-t", "8", "--noSplit", "-o", dst] + opts, check=True,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    print("wrote", dst, os.path.getsize(dst), "bytes", flush=True)
