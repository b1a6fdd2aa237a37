"""K4 `cdr_flags_kernel` (assemble.cu), run from its CUDA source in the emulator, equals the host's restatement of the
reference's --realign predicates (kindel._cdr_inputs, kindel._first_max_base) on adversarial tables: ties among the
clip bases, N-dominant clip weights, zero-depth slots, counts near 2^31 whose sums need 64 bits, clip depths exactly
equal to `tot * decay`, and slot ranges that are not multiples of the block size."""
import numpy as np
import pytest

import emu_harness as E
from kindel_b200 import kindel as K
from kindel_b200.views import BaseCounts

pytestmark = pytest.mark.skipif(not E.available(), reason="needs g++ and the CUDA headers")

DECAYS = (0.0, 0.1, 0.5, 1.0, 0.3, 0.9)
BIG = (1 << 31) - 1


def adversarial_table(seed, n, decay):
    """int32 [19, n]: every slot one of the shapes above (columns 0-4 weights, 5 deletions, 9-13 clip-start and 14-18
    clip-end weights)."""
    rng = np.random.default_rng(seed)
    t = np.zeros((19, n), dtype=np.int64)
    kind = rng.integers(0, 7, n)
    for s in range(n):
        k = int(kind[s])
        if k == 0:    # zero depth everywhere
            continue
        if k == 1:    # small counts, many ties
            t[:6, s] = rng.integers(0, 3, 6)
            t[9:19, s] = rng.integers(0, 3, 10)
        elif k == 2:  # ties among the clip bases' maxima
            m = int(rng.integers(1, 50))
            for c0 in (9, 14):
                t[c0:c0 + 4, s] = rng.choice([m, m, rng.integers(0, m)], 4)
            t[:6, s] = rng.integers(0, 60, 6)
        elif k == 3:  # N-dominant clip weights (N is not clip depth)
            t[9:13, s] = rng.integers(0, 5, 4)
            t[13, s] = int(rng.integers(50, 1000))
            t[14:18, s] = rng.integers(0, 5, 4)
            t[18, s] = int(rng.integers(50, 1000))
            t[:6, s] = rng.integers(0, 20, 6)
        elif k == 4:  # near 2^31: sums need 64 bits
            t[:6, s] = BIG - rng.integers(0, 3, 6)
            t[9:19, s] = BIG - rng.integers(0, 3, 10)
        elif k == 5:  # clip depth exactly tot * decay (and one either side)
            tot = int(rng.integers(1, 1 << 20)) * 10
            t[5, s] = int(rng.integers(0, tot // 10 + 1))
            rest = tot - t[5, s]
            t[:5, s] = np.diff(np.sort(np.concatenate(([0, rest], rng.integers(0, rest + 1, 4)))))
            for c0 in (9, 14):
                cd = int(tot * decay) + int(rng.integers(-1, 2))
                cd = max(cd, 0)
                t[c0:c0 + 4, s] = np.diff(np.sort(np.concatenate(([0, cd], rng.integers(0, cd + 1, 3)))))
                t[c0 + 4, s] = int(rng.integers(0, 3))
        else:         # 2 cd against tot + 1 on either side
            tot = int(rng.integers(0, 1 << 24))
            t[0, s], t[5, s] = tot // 2, tot - tot // 2
            for c0 in (9, 14):
                cd = (tot + 1) // 2 + int(rng.integers(-1, 2))
                t[c0, s] = max(cd, 0)
    assert t.max() <= BIG
    return t.astype(np.int32)


def host_predicates(table, lo, hi, decay):
    """(flags, bases) the way K4 packs them, from the host restatement of the reference's predicates."""
    w = BaseCounts(table[0:5, lo:hi].astype(np.int64))
    dele = table[5, lo:hi].astype(np.int64)
    flags = np.zeros(hi - lo, dtype=np.uint8)
    bases = np.zeros(hi - lo, dtype=np.uint8)
    for d, c0 in enumerate((9, 14)):
        cw = table[c0:c0 + 5, lo:hi].astype(np.int64)
        cd = cw[:4].sum(axis=0)
        _, dominant, extend, b = K._cdr_inputs(w, dele, BaseCounts(cw), cd, decay, 1)
        # (mask_ends = 1 hides the first and last position from region starts; K4 leaves masking to the host)
        dominant[[0, -1]] = cd[[0, -1]] / (w.cols.sum(axis=0) + dele + 1)[[0, -1]] > 0.5
        flags |= (dominant.astype(np.uint8) << (2 * d)) | (extend.astype(np.uint8) << (2 * d + 1))
        code = np.zeros(256, dtype=np.uint8)
        code[np.frombuffer(b"ACGTN", dtype=np.uint8)] = np.arange(5)
        code = code[b]
        assert np.array_equal(b, K._first_max_base(cw))
        bases |= code.astype(np.uint8) << (4 * d)
    return flags, bases


@pytest.mark.parametrize("decay", DECAYS)
def test_k4_emulated_equals_host_predicates(decay):
    seen_dom = seen_ext = 0
    for seed, (n, lo, hi) in enumerate(((1000, 0, 1000), (777, 3, 770), (2048, 255, 1793), (300, 1, 2))):
        t = adversarial_table(seed + int(decay * 100), n, decay)
        want_f, want_b = host_predicates(t, lo, hi, decay)
        got_f, got_b = E.cdr_flags(t, lo, hi, decay)
        bad = np.flatnonzero((got_f != want_f) | (got_b != want_b))
        assert not bad.size, (decay, seed, lo + bad[:5], t[:, lo + bad[:1]].ravel().tolist(), got_f[bad[:3]],
                              want_f[bad[:3]])
        seen_dom += int((want_f & 5).astype(bool).sum())
        seen_ext += int((want_f & 10).astype(bool).sum())
    assert seen_dom > 50 and seen_ext > 50


def test_k4_boundary_cases_are_reached():
    """The table generator really puts clip depths on the comparisons' boundaries."""
    for decay in (0.1, 0.5, 1.0):
        t = adversarial_table(7, 3000, decay).astype(np.int64)
        tot = t[:6].sum(axis=0)
        cd = t[9:13].sum(axis=0)
        assert ((cd == tot * decay) & (tot > 0)).sum() > 20
        assert (2 * cd == tot + 1).sum() + (2 * cd == tot + 2).sum() > 20
        assert (cd + t[13] > 2 ** 32).sum() > 20
