"""Algebraic anchoring of oracle/ringpacking.py (core/rlwe/ring_packing.go) by decryption with real Galois keys, mirroring the
Expand / Pack / Extract-Repack checks of core/rlwe/ring_packing_test.go and their noise bounds (log2 of the standard deviation of
the decryption error): Expand(logGap) leaves coefficient j of the input at X^0 of output j (<= LogN + logGap + 1), Repack puts the
constant coefficient of input k at X^k (<= LogN + 5), and Extract followed by a permuted Repack moves coefficient k to X^perm(k)
(<= LogN + 5). The Galois elements the restatement asks for are exactly the reference's GaloisElementsFor* sets."""
import numpy as np
import pytest

from oracle import ringpacking as ORP
from tests.test_oracle_innersum import _Setup

U64 = np.uint64


def _log2_std(got, want):
    err = np.array([a - b for a, b in zip(got, want)], dtype=np.float64)
    return float(np.log2(np.std(err) + 1e-300))


def _evaluator(S, logN, logGaps=()):
    p = S.params
    ext = S.keys_for(ORP.GaloisElementsForExpand(p, logN))
    rep = S.keys_for(set().union(*[ORP.GaloisElementsForPack(p, g) for g in logGaps]) if logGaps else [])
    return ORP.RingPackingEvaluator(p, ext, rep)


@pytest.mark.parametrize("logN,logGaps", [(8, (0, 3, 8)), (9, (5,)), (10, (8,))])
def test_expand_moves_each_kept_coefficient_to_x0(logN, logGaps):
    S = _Setup(logN, 70 + logN)
    p = S.params
    N = p.N()
    m = S.rng.integers(-(1 << 30), 1 << 30, N)
    for logGap in logGaps:
        for is_ntt in (True, False) if logGap == 3 else (True,):
            ev = _evaluator(S, logN)
            ct = S.encrypt(m, is_ntt)
            cts = ev.Expand(ct, logGap, is_ntt)
            gap = 1 << logGap
            assert sorted(cts) == list(range(0, N, gap))
            assert ev.asked[0] == N + 1 and set(ev.asked) == set(ORP.GaloisElementsForExpand(p, logN))
            for j in list(cts)[:: max(1, len(cts) // 8)]:
                got = S.decrypt(cts[j], S.levelQ, True)            # always NTT domain
                want = [int(m[j])] + [0] * (N - 1)
                assert _log2_std(got, want) <= logN + logGap + 1, (logGap, j, _log2_std(got, want))


@pytest.mark.parametrize("logN", [8, 10])
def test_repack_puts_each_constant_at_its_index(logN):
    S = _Setup(logN, 90 + logN)
    p = S.params
    N = p.N()
    idx = sorted(S.rng.choice(N, 12, replace=False).tolist())
    ms = {k: S.rng.integers(-(1 << 30), 1 << 30, N) for k in idx}        # garbage everywhere but coefficient 0 is zeroed
    ev = _evaluator(S, logN, (logN,))
    out = ev.Repack({k: S.encrypt(ms[k]) for k in idx})
    assert set(ev.asked) <= set(ORP.GaloisElementsForPack(p, logN))
    want = [0] * N
    for k in idx:
        want[k] = int(ms[k][0])
    assert _log2_std(S.decrypt(out, S.levelQ, True), want) <= logN + 5


def test_pack_with_input_gap_and_without_zeroing():
    """Pack(cts, inputLogGap = 2, zeroGarbageSlots = false) of 4 ciphertexts, each encrypting x_k0 + x_k1 X^4 + garbage elsewhere:
    the result holds x_k0 at X^k and x_k1 at X^(4 + k) (the docstring example of ring_packing.go:583-599)."""
    S = _Setup(8, 3)
    p = S.params
    N = p.N()
    ms = {k: S.rng.integers(-(1 << 30), 1 << 30, N) for k in range(4)}
    ev = _evaluator(S, 8, (8,))
    out = ev.Pack({k: S.encrypt(ms[k], False) for k in range(4)}, 2, False, is_ntt=False)
    assert ev.asked == [p.GaloisElement(1 << 5)] * 2 + [p.GaloisElement(1 << 6)]      # pairs (0, 2), (1, 3), then (0, 1)
    got = S.decrypt(out, S.levelQ, True)
    for k in range(4):
        for c in range(0, N, 4):
            assert abs(got[c + k] - int(ms[k][c])) < (1 << 16), (k, c)


@pytest.mark.parametrize("logN", [8, 9])
def test_extract_permute_repack(logN):
    S = _Setup(logN, 50 + logN)
    p = S.params
    N = p.N()
    m = S.rng.integers(-(1 << 30), 1 << 30, N)
    idx = list(range(0, N, N // 16))
    ev = _evaluator(S, logN, (logN,))
    cts = ev.Extract(S.encrypt(m), {i: True for i in idx})
    assert sorted(cts) == idx
    perm = S.rng.permutation(len(idx))
    moved = {idx[perm[n]]: cts[k] for n, k in enumerate(idx)}
    out = ev.Repack(moved)
    want = [0] * N
    for n, k in enumerate(idx):
        want[idx[perm[n]]] = int(m[k])
    assert _log2_std(S.decrypt(out, S.levelQ, True), want) <= logN + 5


def test_quirks_of_pack():
    S = _Setup(8, 1)
    p = S.params
    ev = _evaluator(S, 8, (8,))
    ct = S.encrypt(S.rng.integers(-100, 100, p.N()))
    with pytest.raises(ValueError, match="smaller than inputLogGap"):
        ev.Pack({5: ct}, 8, False)                    # a single input: logGap = LogN, logEnd = 0
    with pytest.raises(ValueError, match="len"):
        ev.Pack({}, 8, True)
    assert ev.Pack({1: ct, 3: ct}, 8, False) is None  # gap 2, logEnd = LogN - 1: slot 0 receives nothing
    ev.asked.clear()
    assert ev.Pack({1: ct}, 8, True) is not None      # b-only at the last step: moves to slot 0
    assert ev.asked[0] == 2 * p.N() - 1              # level 0 (inputLogGap = LogN) uses the conjugation
