"""GPU parity at the edges of the mapping kernels' parameter envelope, against the UNMODIFIED reference (or its stored
results): K1, K2 and K3 stage by stage, bit for bit, at every size where a kernel changes its code path (tests/envelope_data.py
lists the rows and why each sits where it does), with the fast kernels and with the general kernels alone; and the CLI's
PAF at four of them. A context refuses the first sketch size past the general L2 kernel's limit up front."""
import os
import subprocess

import pytest

import envelope_data as ED
import refh
from conftest import have_gpu
from mashmap_b200 import hostlib
from test_gpu_cli import compare_paf, parse
from test_gpu_stages import run_stage_parity

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not have_gpu(), reason="no GPU")]


@pytest.fixture(params=["fast-paths", "general-kernels"])
def kernel_paths(request, monkeypatch):
    """the fast sketch / warp-per-segment L1 / stream L2 kernels (default), or the general sketch / CTA L1 /
    warp-per-candidate L2 kernels alone"""
    if request.param == "general-kernels":
        monkeypatch.setenv("MM_SKETCH_TABLE", "1")
        monkeypatch.setenv("MM_L1_CTA", "1")
        monkeypatch.setenv("MM_L2_GENERAL", "1")
    return request.param


@pytest.fixture(scope="module")
def data(workdir):
    return ED.datasets_by_name(workdir)


RUNS = ED.stage_runs()


@pytest.mark.parametrize("row,which,opts,diag", RUNS, ids=[f"{r[1]}:{' '.join(r[2][:-2])}" for r in RUNS])
def test_stages_at_the_envelope(data, row, which, opts, diag, kernel_paths):
    d = data(which)
    bad = run_stage_parity(d, ["-r", d["ref"], "-q", d["qry"]] + opts, int(opts[opts.index("-s") + 1]),
                           expect_diag=diag if kernel_paths == "fast-paths" else ())
    assert not bad, row


@pytest.mark.parametrize("seg", [5000, 20000])
def test_context_refuses_past_the_general_l2_limit(seg):
    """the general-L2-limit rows sit at the limit: their sketch size makes a context, one more is refused with MM_EINVAL
    before any device memory is taken"""
    from mashmap_b200 import capi

    s = ED.largest_sketch_size(seg)
    capi.Context(kmer_size=19, seg_length=seg, sketch_size=s).close()
    with pytest.raises(capi.MashmapError) as e:
        capi.Context(kmer_size=19, seg_length=seg, sketch_size=s + 1)
    assert e.value.code == capi.MM_EINVAL and "general L2 kernel" in str(e.value), str(e.value)


@pytest.mark.parametrize("which,opts", ED.CLI_RUNS, ids=[ED.cli_name(w, o) for w, o in ED.CLI_RUNS])
def test_cli_paf_at_the_envelope(data, workdir, which, opts):
    """mashmap-b200 prints the reference CLI's PAF (oracle/_ref, or its output stored under tests/golden/envelope)"""
    d = data(which)
    name = ED.cli_name(which, opts)
    stored = os.path.join(ED.PAF_DIR, name + ".paf")
    ref_out, got_out = os.path.join(workdir, f"env_ref_{name}.paf"), os.path.join(workdir, f"env_got_{name}.paf")
    if os.path.exists(refh.REF_BIN):
        subprocess.run([refh.REF_BIN, "-r", d["ref"], "-q", d["qry"], "-t", "8", "-o", ref_out] + opts, check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        assert open(ref_out).read() == open(stored).read(), f"{stored} is stale"
    else:
        ref_out = stored
    p = subprocess.run([hostlib.CLI_PATH, "-r", d["ref"], "-q", d["qry"], "-t", "8", "-o", got_out] + opts,
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    ref_rows, got_rows = parse(ref_out), parse(got_out)
    n_equal, tolerated, problems = compare_paf(ref_rows, got_rows, int(opts[opts.index("-s") + 1]))
    print(f"{name}: reference {len(ref_rows)} lines, ours {len(got_rows)}, equal {n_equal}, tolerated single-fragment "
          f"{tolerated}, problems {len(problems)}")
    for x in problems[:8]:
        print("  ", x)
    assert not problems and n_equal > 0
    if tolerated == 0:
        assert open(got_out).read() == open(ref_out).read()
