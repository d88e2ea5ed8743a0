"""CPU model of the K2 prologue of the ModDown fused with the rescale (lattigo_b200/csrc/keyswitch_fused.cu: ks_add_bcast), evaluated
with correctly rounded IEEE operations on the worst-case operands its stated bound admits and compared with exact integers:
  * q and q_L up to the fp_ok limit ((10 + logN) q < 2^51), in both orders of size, and a q far below q_L,
  * the rescale's value e = cred(r + pHalf, q_L) + q - (pHalf mod q) at its maximum q_L + q - 1, and [P]_q at 1 and q - 1,
  * the ModDown's extension m at the ends of [0, 3q) (ks_ext) and of (-0.66q, 0.66q) (ks_ext_split)."""
import random

import pytest

from tests.test_fp64_arith_model_cpu import fp_canon, fp_mulmod, primes_near_limit


def bcast_prologue(m, e, pm, q):
    """device sequence of ks_add_bcast for one coefficient: m + fp_mulmod(double(e), double([P]_q))"""
    fq, fqinv = float(q), 1.0 / float(q)
    assert e < (1 << 52)                                   # u2d is exact
    t = fp_mulmod(float(e), float(pm), fq, fqinv)
    assert t == int(t) and abs(t) < 0.57 * q, (q, e, pm, t)
    return float(m) + t


@pytest.mark.parametrize("logN", [13, 16])
def test_bcast_prologue_at_its_range_edges(logN):
    rng = random.Random(4)
    qs = primes_near_limit(logN)
    for q in qs:
        for qL in qs:
            if qL == q:
                continue
            emax = qL + q - 1
            es = [emax, emax - 1, q, 1, 0] + [rng.randrange(emax) for _ in range(40)]
            ms = [0, 3 * q - 1, -(int(0.66 * q)), int(0.66 * q)] + [rng.randrange(3 * q) for _ in range(10)]
            for pm in (1, q - 1, rng.randrange(1, q)):
                for e in es:
                    for m in ms:
                        x = bcast_prologue(m, e, pm, q)
                        assert x == int(x) and -2 * q < x < 4 * q, (q, qL, e, m, x)
                        assert abs(x) < 10 * q and (10 + logN) * q < (1 << 51)   # the input range of the forward FP64 transform
                        assert (int(x) - (m + e * pm)) % q == 0
                        assert fp_canon(x, float(q), 1.0 / float(q)) == (m + e * pm) % q
