"""The engine at its own limits (tests/limit_cases.py) on the GPU: every kernel path -- complex reads as pieces or by
atomics, one or seven CTAs per tile, a reused CountTable full of garbage -- gives the C oracle's tables, events and
calls; `bam_to_consensus` with and without --realign equals the host assembly of the oracle's tables; K1q equals the
masking oracle on the quality lattice; and K4 equals the host's --realign predicates on adversarial tables."""
import numpy as np
import pytest

import limit_cases as LC
from oracle import coracle, qoracle
from test_cdr_flags import DECAYS, adversarial_table, host_predicates
from test_limit_cases import GROUPS, batch_of, files  # noqa: F401  (files: the module's fixture)
from test_quality_filters import sam_quals

pytestmark = pytest.mark.gpu


def _device(batch, table=None, repeat=1):
    import torch

    from kindel_b200 import engine

    db = engine.upload(batch)
    for _ in range(repeat):
        counts, events = engine.pileup(db, table=table)
    calls = engine.vote(counts, 1)
    torch.cuda.synchronize()
    return counts.cpu().numpy().copy(), events.cpu().numpy().copy(), calls.cpu().numpy()


@pytest.mark.parametrize("split", ["1", "7"])
@pytest.mark.parametrize("mode", ["atomics", "pieces"])
def test_engine_pileup_on_the_limits(files, monkeypatch, mode, split):  # noqa: F811
    from kindel_b200 import engine

    monkeypatch.setenv("KDL_CX", mode)
    monkeypatch.setenv("KDL_SPLIT", split)
    for name in GROUPS:
        b = batch_of(files, name)
        want_c, want_e = coracle.pileup(b)
        got_c, got_e, calls = _device(b)
        np.testing.assert_array_equal(got_c, want_c, err_msg=name)
        np.testing.assert_array_equal(got_e, want_e, err_msg=name)
        np.testing.assert_array_equal(calls, coracle.vote(want_c, 1), err_msg=name)
        table = engine.CountTable(b.n_slots, engine.require_cuda())
        table.t.fill_(7)                       # garbage everywhere: the first pileup must overwrite / zero it all
        table.dirty, table.dirty_rest = (0, b.n_slots), True
        got_c, got_e, _ = _device(b, table, repeat=2)
        np.testing.assert_array_equal(got_c, want_c, err_msg=name + " (reused table)")
        np.testing.assert_array_equal(got_e, want_e, err_msg=name + " (reused table)")


def test_masked_corpus_equals_the_masking_oracle(files):  # noqa: F811
    for name in GROUPS:
        text = files[name][0]
        plain = batch_of(files, name)
        masked = batch_of(files, name, min_base_quality=LC.MASK_QUAL)
        assert masked.n_masked > 0
        want_c, want_e = qoracle.pileup(plain, sam_quals(text), LC.MASK_QUAL)
        got_c, got_e, calls = _device(masked)
        np.testing.assert_array_equal(got_c, want_c, err_msg=name)
        np.testing.assert_array_equal(got_e, want_e, err_msg=name)
        np.testing.assert_array_equal(calls, coracle.vote(want_c, 1), err_msg=name)


def test_consensus_on_the_limits(files):  # noqa: F811
    from kindel_b200 import bamio
    from kindel_b200 import kindel as K

    for name in GROUPS:
        bam = files[name][2]
        b = bamio.read_alignment(bam)
        counts, events = coracle.pileup(b)
        run = K.PileupRun.from_host_tables(b, counts, coracle.derive(counts), events)
        for realign in (False, True):
            want = K.consensus_from_run(run, coracle.vote(counts, 1), bam, realign=realign)
            got = K.bam_to_consensus(bam, realign=realign)
            assert [(s.name, s.sequence) for s in got.consensuses] == \
                [(s.name, s.sequence) for s in want.consensuses], (name, realign)
            assert got.refs_changes == want.refs_changes, (name, realign)


@pytest.mark.parametrize("decay", DECAYS)
def test_k4_on_the_device(decay):
    import torch

    from kindel_b200 import engine

    for seed, (n, lo, hi) in enumerate(((1000, 0, 1000), (777, 3, 770), (2048, 255, 1793), (300, 1, 2))):
        t = adversarial_table(seed + int(decay * 100), n, decay)
        want_f, want_b = host_predicates(t, lo, hi, decay)
        got_f, got_b = engine.cdr_flags(torch.from_numpy(t).cuda(), lo, hi, decay)
        np.testing.assert_array_equal(got_f, want_f, err_msg="decay %r seed %d" % (decay, seed))
        np.testing.assert_array_equal(got_b, want_b, err_msg="decay %r seed %d" % (decay, seed))
