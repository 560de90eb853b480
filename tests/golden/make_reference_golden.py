"""Writes tests/golden/reference_digests.json from the UNMODIFIED reference (oracle/_ref, built by `make -C oracle ref`
where the reference's sources are): for every command line and data set the GPU tests compare against the reference, the
digests of what the reference computes (tests/golden_ref.py). No GPU needed. Run: python tests/golden/make_reference_golden.py"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import datasets  # noqa: E402
import golden_ref  # noqa: E402
import refh  # noqa: E402
import test_gpu_stages as T  # noqa: E402
from mashmap_b200 import synth  # noqa: E402

assert refh.available(), "oracle/_ref/libmm_ref.so is not built"
wd = tempfile.mkdtemp(prefix="mm_golden_")
out = {"sessions": {}, "fragments": {}, "sketch_random_set": {}, "sketch_degenerate": {}, "sketch_every_k": {}}
sets = {"random": datasets.make_random_set(wd), "panel": datasets.make_panel_set(wd), "asm": datasets.make_assembly_set(wd),
        "hifi": datasets.make_hifi_set(wd), "big": datasets.make_big_random_set(wd), "rep": datasets.make_repeat_set(wd)}
# tests/test_gpu_stages.py: run_stage_parity and test_packed_input_equals_text_input
stage_runs = [("random", ["-s", "5000", "--pi", "85", "-t", "4"]), ("random", ["-s", "5000", "--pi", "95", "--dense", "-t", "4"]),
              ("panel", ["-s", "5000", "--pi", "85", "-t", "4"]), ("panel", ["-s", "2000", "--pi", "90", "-J", "25", "--noHgFilter", "-t", "4"]),
              ("panel", ["-s", "5000", "--pi", "85", "--kmerThreshold", "5", "-t", "4"]),
              ("asm", ["-s", "10000", "--pi", "90", "-f", "one-to-one", "-t", "4"]),
              ("hifi", ["-s", "5000", "--pi", "95", "-J", "20", "-f", "one-to-one", "-t", "4"]),
              ("big", ["-s", "5000", "--pi", "95", "--dense", "-t", "8"]), ("big", ["-s", "5000", "--pi", "85", "-J", "220", "-t", "8"]),
              ("rep", ["-s", "5000", "--pi", "85", "-t", "4"]), ("rep", ["-s", "5000", "--pi", "85", "--noHgFilter", "-t", "4"])]
for name, opts in stage_runs:
    d = sets[name]
    args = ["-r", d["ref"], "-q", d["qry"]] + opts
    key = golden_ref.key_of(args, d)
    R = refh.RefSession(args)
    out["sessions"][key] = golden_ref.session_digests(R)
    lens = [len(r) for r in d["reads"]]
    ridx, start, length = synth.split_segments(lens, R.p.segLength, R.p.kmerSize)
    out["fragments"][key] = [golden_ref.reference_fragment_digest(
        R.map_fragment(d["rnames"][ridx[i]], d["reads"][ridx[i]][start[i] : start[i] + length[i]], full_len=lens[ridx[i]],
                       seq_counter=int(ridx[i]))) for i in range(len(ridx))]
    R.close()
    print(key, len(ridx), "fragments", flush=True)
# tests/test_gpu_index_build.py
index_runs = [(datasets.make_random_set(wd, tag="ixr"), ["-s", "5000", "--pi", "85", "-t", "4"]),
              (datasets.make_panel_set(wd, tag="ixp"), ["-s", "5000", "--pi", "85", "--kmerThreshold", "5", "-t", "4"]),
              (datasets.make_big_random_set(wd, tag="ixb", n_contigs=4, contig_len=1_000_000, n_reads=2), ["-s", "5000", "--pi", "95", "--dense", "-t", "8"])]
for d, opts in index_runs:
    args = ["-r", d["ref"], "-q", d["qry"]] + opts
    R = refh.RefSession(args)
    out["sessions"][golden_ref.key_of(args, d)] = golden_ref.session_digests(R)
    R.close()


def sketch_digests(reads, seg_length, k, s):
    ridx, start, length = synth.split_segments([len(r) for r in reads], seg_length, k)
    return [golden_ref.sketch_digest(refh.sketch_sequence(reads[ridx[i]][start[i] : start[i] + length[i]], k, s, seq_id=int(ridx[i])))
            for i in range(len(ridx))]


for k, s in [(19, 130), (16, 40), (21, 250), (32, 17)]:
    out["sketch_random_set"][f"k{k} s{s}"] = sketch_digests(sets["random"]["reads"], 5000, k, s)
out["sketch_degenerate"]["k19 s100"] = [golden_ref.sketch_digest(refh.sketch_sequence(q, 19, 100, seq_id=i))
                                        for i, q in enumerate(T.degenerate_sequences())]
for k in range(8, 33):
    out["sketch_every_k"][f"k{k} s60"] = sketch_digests(T.every_k_subset(sets["random"])["reads"], 3000, k, 60)
# tests/test_args_cpu.py
import test_args_cpu as TA  # noqa: E402

out["parameters"], out["reference_size"] = {}, {}
d = datasets.make_panel_set(wd, tag="args", n_strains=2, chrom_len=40_000)
for opts in TA.OPTION_SETS:
    for with_query in (True, False):
        args = ["-r", d["ref"]] + (["-q", d["qry"]] if with_query else []) + ["-t", "2"] + opts
        out["parameters"][golden_ref.key_of(args, d)] = TA.reference_parameters(args, d)
for size in (2**31 - 1000, 2**31 + 1000, 3_100_000_000, 5_000_000_000, 2**32 + 4096):
    f = os.path.join(wd, "big.fa")
    with open(f, "wb") as fh:
        fh.write(b">c\nACGT\n")
        fh.truncate(size)
    out["reference_size"][str(size)] = TA.reference_size_and_sketch(["-r", f, "-q", f, "-s", "5000", "--pi", "85"], size)
    os.remove(f)
json.dump(out, open(golden_ref.PATH, "w"), separators=(",", ":"), sort_keys=True)
print("wrote", golden_ref.PATH, os.path.getsize(golden_ref.PATH), "bytes")
