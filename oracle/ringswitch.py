"""CPU restatement of the generic key switch with ring-degree switching (reference, pure Go):

    SwitchCiphertextRingDegreeNTT                 core/rlwe/element.go:250-287
    SwitchCiphertextRingDegree                    core/rlwe/element.go:293-312
    Evaluator.ApplyEvaluationKey                  core/rlwe/evaluator_evaluationkey.go:36-107
    ExtendBasisSmallNormAndCenterNTTMontgomery    core/rlwe/utils.go:250-284
    KeyGenerator.GenEvaluationKey (any degrees)   core/rlwe/keygenerator.go:261-285

TEST INFRASTRUCTURE ONLY, like the rest of oracle/: built on oracle/oracle.py's rings and Evaluator.GadgetProduct and on
oracle/encryptor.py's gen_evaluation_key. The downward NTT-domain switch is restated literally: per row an INTT at the large degree,
every gap-th coefficient, and NTTStandard (NTTConjugateInvariant) at the small degree called with the LARGE ring's RootsForward.
`block_average` is the one-pass form the device uses (DESIGN 3.4); tests/test_oracle_ringswitch.py checks that the two agree.

Conventions: ciphertexts are pairs [c0, c1] of (rows, degree) uint64 arrays; `is_ntt` is the reference's MetaData.IsNTT. Secret
keys are (rows, degree) NTT + Montgomery arrays, as rlwe.SecretKey.Value.Q (and .P) hold them."""
from __future__ import annotations

import numpy as np

from . import encryptor as OE
from . import oracle as O

U64 = np.uint64


def _ntt_with_table(sub: O.SubRing, row: np.ndarray, n: int):
    """ring.NTTStandard / NTTConjugateInvariant(row, row, n, s.Modulus, s.MRedConstant, s.BRedConstant, s.RootsForward) with the
    SubRing `sub` of the large degree."""
    f = O.lib().lo_ntt if sub.Type == "Standard" else O.lib().lo_ntt_ci
    f(O._ptr(row), O._ptr(row), n, sub.Modulus, sub.MRedConstant, O._ptr(sub.brc), O._ptr(sub.RootsForward))


def SwitchCiphertextRingDegreeNTT(ctIn, ringQLargeDim, opOut):
    NIn, NOut = ctIn[0].shape[1], opOut[0].shape[1]
    if NIn > NOut:
        gap = NIn // NOut
        buff = np.empty(NIn, dtype=U64)
        for i in range(len(opOut)):
            for j in range(opOut[i].shape[0]):
                tmpIn = np.ascontiguousarray(ctIn[i][j])         # IndexError where the reference's loop panics (opOut has more rows)
                s = ringQLargeDim.SubRings[j]
                s.INTT(tmpIn, buff)
                tmpOut = np.ascontiguousarray(buff[::gap])
                _ntt_with_table(s, tmpOut, NOut)
                opOut[i][j] = tmpOut
    else:
        for i in range(len(opOut)):
            O.MapSmallDimensionToLargerDimensionNTT(ctIn[i], opOut[i])


def SwitchCiphertextRingDegree(ctIn, opOut):
    NIn, NOut = ctIn[0].shape[1], opOut[0].shape[1]
    gapIn, gapOut = NOut // NIn, 1
    if NIn > NOut:
        gapIn, gapOut = 1, NIn // NOut
    for i in range(len(opOut)):
        for j in range(opOut[i].shape[0]):
            tmp1 = ctIn[i][j]                                    # IndexError where the reference panics
            opOut[i][j][0:NOut:gapIn] = tmp1[0:NIn:gapOut]


def block_average(A: np.ndarray, n: int, q: int) -> np.ndarray:
    """out[j] = gap^-1 * sum_{u < gap} A[j gap + u] mod q for one row A of the large degree (python integers, exact)."""
    gap = A.shape[0] // n
    s = A.astype(object).reshape(n, gap).sum(axis=1)
    ginv = pow(gap, -1, q)
    return np.array([int(v) * ginv % q for v in s], dtype=U64)


def _applyEvaluationKey(ev: O.Evaluator, level, ctIn, evk, opOut, is_ntt):
    """:99-107"""
    N = ev.params.N()
    ctTmp = [np.zeros((level + 1, N), dtype=U64) for _ in range(2)]
    ev.GadgetProduct(level, np.ascontiguousarray(ctIn[1][: level + 1]), evk, ctTmp, is_ntt)
    ringQ = ev.params.ringQ.AtLevel(level)
    out0 = np.empty((level + 1, N), dtype=U64)
    ringQ.Add(np.ascontiguousarray(ctIn[0][: level + 1]), ctTmp[0], out0)
    opOut[0][: level + 1] = out0
    opOut[1][: level + 1] = ctTmp[1]


def ApplyEvaluationKey(ev: O.Evaluator, ctIn, evk: O.GadgetCiphertext, opOut, is_ntt: bool = True):
    """:36-97. ev: the evaluator of the large degree. opOut is written in place (rows 0..min(levels) and, going up, the map)."""
    level = min(ctIn[0].shape[0], opOut[0].shape[0]) - 1
    ringQ = ev.params.ringQ.AtLevel(level)
    NIn, NOut = ctIn[0].shape[1], opOut[0].shape[1]
    if NIn < NOut:
        if NOut != ringQ.N():
            raise ValueError("cannot ApplyEvaluationKey: opOut ring degree does not match evaluator params ring degree")
        if is_ntt:
            SwitchCiphertextRingDegreeNTT(ctIn, None, opOut)
        else:
            SwitchCiphertextRingDegree(ctIn, opOut)
        _applyEvaluationKey(ev, level, opOut, evk, opOut, is_ntt)
    elif NIn > NOut:
        if NIn != ringQ.N():
            raise ValueError("cannot ApplyEvaluationKey: ctIn ring degree does not match evaluator params ring degree")
        ctTmp = [np.zeros((level + 1, NIn), dtype=U64) for _ in range(2)]
        _applyEvaluationKey(ev, level, ctIn, evk, ctTmp, is_ntt)
        if is_ntt:
            SwitchCiphertextRingDegreeNTT(ctTmp, ringQ, opOut)
        else:
            SwitchCiphertextRingDegree(ctTmp, opOut)
    else:
        _applyEvaluationKey(ev, level, ctIn, evk, opOut, is_ntt)


def ExtendBasisSmallNormAndCenterNTTMontgomery(rQ: O.Ring, rP: O.Ring, polQ, polP):
    rQ = rQ.AtLevel(0)
    buff = np.empty((1, rQ.N()), dtype=U64)
    rQ.INTT(np.ascontiguousarray(polQ[:1]), buff)
    rQ.IMForm(buff, buff)
    Q = rQ.SubRings[0].Modulus
    QHalf = Q >> 1
    P = rP.ModuliChain()[: rP.Level() + 1]
    c = buff[0].astype(object)
    neg = c > QHalf
    mag = np.where(neg, Q - c, c)
    for i, pi in enumerate(P):
        polP[i] = np.where(neg, pi - mag, mag).astype(U64)
    rP.NTT(polP, polP)
    rP.MForm(polP, polP)


def GenEvaluationKey(params: O.Parameters, skIn, skOut, rng, pw2=0, sigma=3.2) -> O.GadgetCiphertext:
    """:261-285 at the maximum levels of `params` (the large degree), with fresh uniform / Gaussian samples from rng.
    skIn: (rows, n_in) NTT + Montgomery rows of SecretKey.Value.Q; skOut: (rows, n_out) rows of SecretKey.Value.Q."""
    ringQ, ringP = params.ringQ, params.ringP
    N = params.N()
    nQ = len(params.qi)
    nP = len(params.pi)
    buffSkOut = np.zeros((nQ + nP, N), dtype=U64)
    outQ = np.zeros((nQ, N), dtype=U64)
    O.MapSmallDimensionToLargerDimensionNTT(skOut, outQ)
    buffSkOut[:nQ] = outQ
    if nP:
        polP = np.zeros((nP, N), dtype=U64)
        ExtendBasisSmallNormAndCenterNTTMontgomery(ringQ, ringP.AtLevel(nP - 1), outQ, polP)
        buffSkOut[nQ:] = polP
    buffSkIn = np.zeros((nQ, N), dtype=U64)
    O.MapSmallDimensionToLargerDimensionNTT(skIn, buffSkIn)
    levelOut = skOut.shape[0] - 1
    ext = np.zeros((levelOut + 1, N), dtype=U64)
    ExtendBasisSmallNormAndCenterNTTMontgomery(ringQ, ringQ.AtLevel(levelOut), buffSkIn, ext)
    buffSkIn[: levelOut + 1] = ext
    n = params.BaseRNSDecompositionVectorSize(params.MaxLevelQ(), params.MaxLevelP())
    sizes = params.BaseTwoDecompositionVectorSize(params.MaxLevelQ(), params.MaxLevelP(), pw2)[:n]
    mods = params.qi + params.pi
    a = [[np.stack([rng.integers(0, int(m), N, dtype=U64) for m in mods]) for _ in range(sizes[i])] for i in range(n)]
    e = [[np.rint(rng.normal(0, sigma, N)).astype(np.int64) for _ in range(sizes[i])] for i in range(n)]
    return OE.gen_evaluation_key(params, buffSkIn, buffSkOut, a, e, pw2)
