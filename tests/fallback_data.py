"""Data of tests/test_gpu_fallbacks.py that has stored reference results (tests/golden/make_fallback_golden.py): repeat
sets whose exact tandem array has 16, 17 and 24 copies, mapped without the HG filter."""
import datasets

TANDEM_COPIES = (16, 17, 24)


def tandem_set(workdir, n):
    return datasets.make_repeat_set(workdir, tag=f"rep{n}", tandem_copies=n)


def tandem_args(d):
    return ["-r", d["ref"], "-q", d["qry"], "-s", "5000", "--pi", "85", "--noHgFilter", "-t", "4"]
