"""bin/rsem-for-ebseq-calculate-clustering-info against the reference tool (oracle/_ref/rsem-for-ebseq-calculate-
clustering-info, built by oracle/ebseq.mk): stdout and the output file must be byte-identical.  Where the reference
binary is not built, its stdout and the output's SHA-256 come from tests/golden/reference/ebseq_*.tar.xz
(rsem_files.reference_run; RSEM_B200_RECORD_REFERENCE=1 rewrites them).

Cases: the FASTA quirks (CRLF, IUPAC and lowercase letters, empty entries), duplicate sequences, repeats inside one
transcript only, shared N runs, transcripts of length k and k - 1, k from 1 to 150 on one small family-structured
transcriptome, and a few-Mb one at k = 25 and 100.  Through the C ABI (K9) against the sort-based C restatement:
runs forced into several passes by a small device budget, and a 1-bit fingerprint, so that most probes verify."""
import hashlib
import os

import numpy as np
import pytest

import clustering_info as ci

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("key", sorted(ci.DEVICE_CASES))
def test_executable_matches_reference(built, tmp_path, key):
    k, make = ci.DEVICE_CASES[key]
    data = make()
    ref = ci.write_case(str(tmp_path / "ref"), data)
    ours = ci.write_case(str(tmp_path / "ours"), data)
    r = ci.reference(key, ref, k)
    assert r.returncode == 0
    p = ci.run(ci.BIN, ours, k)
    assert p.returncode == 0, p.stderr
    assert p.stdout == r.stdout
    assert hashlib.sha256(open(os.path.join(ours, ci.OUT), "rb").read()).hexdigest() == r.digests[ci.OUT]


@pytest.fixture(scope="module")
def family():
    names, seqs = ci.family_transcriptome(400_000, 77, iupac=True)
    _, off, bases, _ = ci.load_ref(ci.to_fasta(names, seqs))
    return off, bases


@pytest.fixture(scope="module")
def ctx(built):
    import rsem_b200
    with rsem_b200.Context(0) as c:
        yield c


@pytest.mark.parametrize("k", [1, 25, 33, 64, 150])
def test_capi_matches_restatement(ctx, family, k):
    off, bases = family
    counts, st = ctx.kmer_shared(k, off, bases)
    assert st.passes == 1 and st.positions == int(ci.eff_lengths(k, off).sum())
    assert np.array_equal(counts, ci.oracle_counts(k, off, bases))


@pytest.mark.parametrize("k,passes", [(25, 2), (25, 5), (64, 7), (33, 2)])
def test_forced_passes(ctx, family, k, passes):
    """budget = input + 12 bytes x 2 positions / passes: the k-mers split over that many passes of one table"""
    off, bases = family
    want = ci.oracle_counts(k, off, bases)
    _, st = ctx.kmer_shared(k, off, bases)
    budget = st.input_bytes + 12 * (2 * st.positions // passes)
    counts, st = ctx.kmer_shared(k, off, bases, max_device_bytes=budget)
    assert st.passes == passes if passes == 2 else st.passes >= passes
    assert st.table_bytes + st.input_bytes <= budget
    assert np.array_equal(counts, want)


@pytest.mark.parametrize("k,passes", [(5, 1), (33, 1), (33, 3)])
def test_small_fingerprint(ctx, family, k, passes):
    """1 fingerprint bit: half the probes past a k-mer's slot go through the base-by-base verification"""
    off, bases = family
    want = ci.oracle_counts(k, off, bases)
    _, st = ctx.kmer_shared(k, off, bases)
    budget = st.input_bytes + 12 * (2 * st.positions // passes) if passes > 1 else 0
    counts, st = ctx.kmer_shared(k, off, bases, max_device_bytes=budget, fingerprint_bits=1)
    assert st.passes >= passes
    assert np.array_equal(counts, want)


def test_no_positions(ctx):
    """every transcript shorter than k: zero counts, no device work"""
    off = np.array([0, 10, 25], np.uint64)
    counts, st = ctx.kmer_shared(26, off, np.zeros(25, np.uint8))
    assert st.passes == 0 and st.positions == 0 and not counts.any()
