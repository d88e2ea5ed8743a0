"""lgpu_bgv_polynomial_evaluate against the literal op-by-op oracle (tests/bgv_polyeval_oracle.py), bit for bit, with the output level
and scale, for the BGV (tensorStandard) and BFV (tensorScaleInvariant) evaluators:
- N = 2^10 to 2^12 with every polynomial case, batch 1 and 3, at the top level and at the lowest level the reference accepts;
- one batch larger than batch_chunk(), so that the runner crosses sub-batches;
- BGV_N15QP880 (t = 0x10001, level 19, batch 16, degrees 15 and 63);
- N = 2^16 BFV on 12 Q + 4 P limbs;
- a run entirely on the device: BGVEncoder.Encode, encryption, Evaluate, decryption with ring ops and Decode give p(m) mod t."""
import os

import numpy as np
import pytest

from lattigo_b200 import bgv_polyeval as BPE
from lattigo_b200 import params as presets
from oracle import encryptor as ENC
from oracle import oracle as O
from tests import bgv_oracle as B
from tests import bgv_polyeval_cases as C
from tests import bgv_polyeval_oracle as BP
from tests import helpers as H

pytestmark = pytest.mark.gpu


class Device:
    """One context with a uniform relinearization key, the device evaluators and the oracle ones."""

    def __init__(self, logN, q, p, t, seed):
        import lattigo_b200 as lb
        self.N, self.q, self.p, self.t = 1 << logN, list(q), list(p), int(t)
        self.params = O.Parameters(logN, self.q, self.p)
        self.qmul = B.qmul_moduli(logN, self.q)
        self.rng = np.random.default_rng(seed)
        self.rlk_o = H.random_gadget_ciphertext(self.params, len(q) - 1, len(p) - 1, self.rng)
        self.ctx = lb.Context(logN, self.q, self.p)
        self.rlk = lb.GadgetCiphertext(self.ctx, self.rlk_o.data, len(q) - 1, len(p) - 1)
        self.pev = {}
        for si in (False, True):
            ev = lb.BGVEvaluator(self.ctx, self.t, self.qmul, self.rlk, scale_invariant=si)
            self.pev[si] = lb.BGVPolynomialEvaluator(ev)

    def cts(self, level, batch):
        return np.stack([np.stack([H.rand_poly(self.q[: level + 1], self.N, self.rng) for _ in range(2)]) for _ in range(batch)])

    def oracle(self, si, ct, scale, coeffs, target, odd, even):
        pe = BP.PolyEvaluator(self.params, self.rlk_o, self.t, self.qmul, si)
        return pe.Evaluate(BP.P.Ct([ct[0], ct[1]], scale), BP.new_polynomial(coeffs, odd, even), target)

    def check(self, si, cts, coeffs, odd=True, even=True, scale=1, target=1, idx=None):
        out, level, sc = self.pev[si].Evaluate(self.ctx.to_device(cts), scale, coeffs, target, odd, even)
        out = self.ctx.to_host(out)
        for k in (range(len(cts)) if idx is None else idx):
            r = self.oracle(si, cts[k], scale, coeffs, target, odd, even)
            assert (level, sc) == (r.Level(), int(r.Scale))
            assert np.array_equal(out[k], np.stack(r.Value)), k


def _lowest(d, coeffs, si, odd, even):
    L = len(d.q) - 1
    ok = [lv for lv in range(L + 1) if _plans(d, lv, coeffs, si, odd, even)]
    return min(ok)


def _plans(d, lv, coeffs, si, odd, even):
    try:
        BPE.plan(d.q, d.t, lv, 1, coeffs, 1, si, odd, even)
        return True
    except ValueError:
        return False


@pytest.mark.parametrize("logN", [10, 11, 12])
def test_small_rings_every_case(logN):
    q, p = O.gen_moduli(logN + 1, [55] + [45] * 9, [60, 60])
    t = 0xffc001 if logN == 10 else 0x10001
    d = Device(logN, q, p, t, seed=logN)
    L = len(q) - 1
    cts = d.cts(L, 3)
    for name, (coeffs, odd, even) in C.cases(t).items():
        for si in (False, True):
            batch = 3 if name in ("d15", "x2") else 1
            d.check(si, cts[:batch], coeffs, odd, even)
            low = _lowest(d, coeffs, si, odd, even)
            d.check(si, np.ascontiguousarray(cts[:1, :, : low + 1]), coeffs, odd, even)
    for si in (False, True):                                   # scale and target scale other than 1
        d.check(si, cts[:1], C.cases(t)["d7"][0], scale=5, target=12345)


def test_batch_larger_than_batch_chunk():
    q, p = O.gen_moduli(11, [55] + [45] * 5, [60])
    d = Device(10, q, p, 0x10001, seed=2)
    batch = int(os.environ.get("LGPU_BATCH_CHUNK", "64")) + 3          # batch_chunk() + 3
    cts = d.cts(len(q) - 1, batch)
    coeffs = C.cases(d.t)["d7"][0]
    for si in (False, True):
        d.check(si, cts, coeffs, idx=(0, batch - 4, batch - 3, batch - 1))


@pytest.fixture(scope="module")
def n15():
    sp = presets.PRESETS["BGV_N15QP880"]
    return Device(sp["logN"], sp["Q"], sp["P"], sp["T"], seed=15)


@pytest.mark.parametrize("degree", [15, 63])
def test_n15qp880_level19_batch16(n15, degree):
    d = n15
    cts = d.cts(19, 16)
    coeffs = C.cases(d.t)["d%d" % degree][0]
    for si in (False, True):
        d.check(si, cts, coeffs, idx=(0, 15))


def test_pn16_bfv_12q_4p():
    sp = presets.PRESETS["CKKS_PN16QP1761"]
    d = Device(16, sp["Q"][:12], sp["P"], 0x10001, seed=16)
    d.check(True, d.cts(11, 2), C.cases(d.t)["d3"][0], idx=(0, 1))


def test_device_end_to_end():
    """Encode, encrypt (EncryptZeroSk + Add), Evaluate, decrypt with ring ops and Decode: p(m) mod t slot-wise, BGV and BFV."""
    import torch
    import lattigo_b200 as lb
    logN, t, batch = 11, 0x10001, 2
    q, p = O.gen_moduli(logN + 1, [55] + [45] * 9, [60, 60])
    L = len(q) - 1
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    enc = lb.BGVEncoder(ctx, t)
    N, n = ctx.N, enc.MaxSlots()
    rng = np.random.default_rng(21)
    s = rng.integers(-1, 2, N)
    rlk = lb.GadgetCiphertext(ctx, H.gen_switching_key(params, C.Toy._sq(s), s, rng).data, L, len(p) - 1)
    sk = ENC.small_rows(s, params.qi)
    params.ringQ.NTT(sk, sk); params.ringQ.MForm(sk, sk)
    d_sk = ctx.to_device(sk)
    m = rng.integers(0, t, (batch, n), dtype=np.int64)
    pt = enc.Encode(m, L)
    c1 = ctx.to_device(np.stack([np.stack([rng.integers(0, qi, N, dtype=np.uint64) for qi in q]) for _ in range(batch)]))
    e = torch.from_numpy(np.rint(rng.normal(0, 3.2, (batch, N))).astype(np.int64)).cuda()
    c0 = lb.encryptor.Encryptor(ctx).EncryptZeroSk(L, -1, d_sk, c1, e, True, False)
    ctx.ringQ.AtLevel(L).Add(c0, pt, c0)
    ct = torch.stack([c0, c1], dim=1).contiguous()
    coeffs = C.cases(t)["d15"][0]
    for si in (False, True):
        pe = lb.BGVPolynomialEvaluator(lb.BGVEvaluator(ctx, t, B.qmul_moduli(logN, q), rlk, scale_invariant=si))
        out, lv, sc = pe.Evaluate(ct, 1, coeffs, 1)
        rl = ctx.ringQ.AtLevel(lv)
        skb = d_sk[: lv + 1].unsqueeze(0).expand(batch, -1, -1).contiguous()
        x = out[:, 0].clone()
        rl.MulCoeffsMontgomeryThenAdd(out[:, 1].contiguous(), skb, x)
        got = enc.Decode(x, sc).cpu().numpy()
        want = np.array([[C.eval_poly_mod(coeffs, int(v), t) for v in row] for row in m])
        assert np.array_equal(got, want), si
        assert sc == 1 and (lv == L if si else lv < L)
