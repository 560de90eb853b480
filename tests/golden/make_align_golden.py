"""Writes tests/golden/align/: the mapping file the reference mapper prints with --legacy for the ONT-like reads of
tests/align_cases.py, and the sha256 of the unmodified reference aligner's output for every case. Needs oracle/_ref
(mashmap_ref, mashmap_align_ref). Usage: python tests/golden/make_align_golden.py"""
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import align_cases as AC  # noqa: E402
import align_data as AD  # noqa: E402


def main():
    os.makedirs(AC.GOLDEN, exist_ok=True)
    d = tempfile.mkdtemp()
    try:
        AC.write_inputs(d)
        out = os.path.join(d, "legacy.map")
        subprocess.run([AD.MAP_REF_BIN, "-r", os.path.join(d, "ref.fa"), "-q", os.path.join(d, "reads.fa"), "--pi", "80",
                        "--legacy", "-t", "4", "-o", out], check=True, capture_output=True, cwd=d)
        shutil.copy(out, AC.MAPPED)
        digests = {}
        for name in AC.CASES:
            o = os.path.join(d, name + ".sam")
            subprocess.run([AD.ALIGN_REF_BIN] + AC.case_args(d, name) + ["-o", o], check=True, capture_output=True, cwd=d)
            data = open(o, "rb").read()
            digests[name] = {"sha256": hashlib.sha256(data).hexdigest(), "lines": data.count(b"\n")}
            print(name, digests[name])
        with open(os.path.join(AC.GOLDEN, "reference_outputs.json"), "w") as f:
            json.dump(digests, f, indent=1, sort_keys=True)
    finally:
        shutil.rmtree(d)


if __name__ == "__main__":
    main()
