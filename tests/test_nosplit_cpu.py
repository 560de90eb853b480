"""No GPU: the checkers of the long-fragment tests (tests/test_gpu_nosplit.py). The oracle's sketchSequence restatement on
fragments longer than a segment equals the unmodified reference (oracle/_ref, where built) and the reference's stored
digests (tests/golden/nosplit_digests.json)."""
import pytest

import golden_ref
import nosplit_data as ND
import oracle_py
import refh

pytestmark = pytest.mark.skipif(not oracle_py.available(), reason="oracle/libmm_oracle.so not built")


@pytest.mark.parametrize("k,s", ND.SKETCH_CASES)
def test_oracle_long_fragment_sketch_equals_stored_reference(k, s):
    seqs = ND.long_sequences(k)
    got = [golden_ref.sketch_digest(oracle_py.sketch_sequence(q, k, s, seq_id=i)) for i, q in enumerate(seqs)]
    assert got == ND.get("sketch_long", f"k{k} s{s}")


@pytest.mark.skipif(not refh.available(), reason="oracle/_ref not built")
@pytest.mark.parametrize("k,s", ND.SKETCH_CASES)
def test_oracle_long_fragment_sketch_equals_reference(k, s):
    for i, q in enumerate(ND.long_sequences(k)):
        a, b = oracle_py.sketch_sequence(q, k, s, seq_id=i), refh.sketch_sequence(q, k, s, seq_id=i)
        assert a.tobytes() == b.tobytes(), (i, len(q))


@pytest.mark.parametrize("which,opts", ND.STAGE_RUNS)
def test_oracle_whole_query_stages_equal_reference(workdir, which, opts):
    """the oracle's windowLen > 0 code (computeL1CandidateRegions / computeL2MappedRegions with hash_to_freq) on every
    query of the data set mapped as one fragment: equal to the reference's stages (computed where oracle/_ref is built,
    otherwise stored); the index comes from the reference, or from the product's host builder checked against the
    reference's stored digests"""
    d = ND.datasets_by_name(workdir)[which]()
    args = ["-r", d["ref"], "-q", d["qry"]] + opts
    key = golden_ref.key_of(args, d)
    if refh.available():
        R = refh.RefSession(args)
        contig_len, names = R.contig_len, R.contig_names
    else:
        R = golden_ref.ProductSession(args)
        assert golden_ref.session_digests(R) == golden_ref.get("sessions", key)
        contig_len, names = [len(c) for c in d["genome"]], list(d["names"])
    try:
        O = oracle_py.Oracle(params=R.p)
        keys, offs, pts, fr = R.lookup()
        O.set_index(R.index(), keys, offs, pts, fr, contig_len, names)
        ridx, lens = ND.whole_reads(d, R.p.kmerSize)
        got = [golden_ref.reference_fragment_digest(O.map_fragment(d["reads"][i], seq_counter=int(i), full_len=int(n)))
               for i, n in zip(ridx, lens)]
        O.close()
        if refh.available():
            want = [golden_ref.reference_fragment_digest(R.map_fragment(d["rnames"][i], d["reads"][i], full_len=int(n), seq_counter=int(i)))
                    for i, n in zip(ridx, lens)]
            ND.check_stored("fragments", key, want)
        else:
            want = ND.get("fragments", key)
        assert got == want
    finally:
        R.close()
