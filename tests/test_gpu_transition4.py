"""The 4-state transition-matrix kernel (k_transition4: every instance with S <= 4 and at most 32 categories).

Each case checks getTransitionMatrix of every branch against a numpy restatement of BaseSubstitutionModel.java:206-241 and
ComplexColtEigenSystem.java:71-139, then runs full evaluations against the oracle. The evaluations read the other copies
the kernel writes: the spectra (eigen-form walk, real systems), the [j][CP][i] block (matrix-form walk) and the tensor
walk's Mpad / MTg copies (B200_WALK_VARIANT=2, C in {1, 2, 4, 8}).
"""
import numpy as np
import pytest

import helpers as H
from beast_mcmc_b200 import beagle
from harness import evomodel as em, treedatalikelihood as tdl

pytestmark = pytest.mark.gpu

GPU = beagle.BeagleFactory.loadBeagleInstance
EPS = np.finfo(np.float64).eps
REL = 1e-10
LENGTHS = np.array([0.0, 1e-9, 1e-3, 0.1, 1.0, 7.5, 50.0])


class _ComplexModel(em.SubstitutionModel):
    """A non-reversible generator with a complex-conjugate eigenvalue pair, in the real block form BEAST's
    ComplexColtEigenSystem passes: rows k, k+1 of a pair hold Re/Im of the eigenvector, Eval = real parts || imaginary parts."""

    def __init__(self, S, seed):
        rng = np.random.default_rng(seed)
        q = rng.uniform(0.05, 0.3, (S, S))
        for i in range(S):
            q[i, (i + 1) % S] = 3.0                     # a strong cycle: complex eigenvalues
        np.fill_diagonal(q, 0.0)
        np.fill_diagonal(q, -q.sum(axis=1))
        lam, v = np.linalg.eig(q)
        assert (np.abs(lam.imag) > 1e-3).any()
        evec, evr, evi, col, used = np.zeros((S, S)), np.zeros(S), np.zeros(S), 0, set()
        for k in range(S):
            if k in used:
                continue
            used.add(k)
            if abs(lam[k].imag) < 1e-12:
                evec[:, col] = v[:, k].real
                evr[col] = lam[k].real
                col += 1
            else:
                m = next(m for m in range(S) if m not in used and abs(lam[m] - np.conj(lam[k])) < 1e-9)
                used.add(m)
                evec[:, col], evec[:, col + 1] = v[:, k].real, v[:, k].imag
                evr[col] = evr[col + 1] = lam[k].real
                evi[col], evi[col + 1] = lam[k].imag, -lam[k].imag
                col += 2
        w, u = np.linalg.eig(q.T)                        # stationary distribution: root frequencies
        pi = np.abs(u[:, np.argmin(np.abs(w))].real)
        super().__init__(np.ones(S * (S - 1) // 2), pi / pi.sum())
        self.q = q
        self._eigen = em.EigenDecomposition(evec, np.linalg.inv(evec), np.concatenate([evr, evi]))

    def canReturnComplexDiagonalization(self):
        return True

    def infinitesimalMatrix(self):
        return self.q


def _real_model(S, seed):
    if S == 4:
        return em.GTR(1.0, 4.0, 0.7, 1.2, 5.0, 1.0, np.array([0.30, 0.22, 0.24, 0.24]))
    rng = np.random.default_rng(seed)
    return em.SubstitutionModel(rng.uniform(0.2, 3.0, S * (S - 1) // 2), rng.dirichlet(np.full(S, 5.0)))


def _restated(evec, ievc, evals, d):
    """P(d) with the reference's block rule and abs(), and sum_k |Evec[i][k]| |iexp[k][j]| (the scale of the rounding)."""
    S = evec.shape[0]
    complex_form = evals.shape[0] == 2 * S
    ec, es, pt = np.zeros(S), np.zeros(S), np.arange(S)
    k = 0
    while k < S:
        if not complex_form or evals[S + k] == 0.0:
            ec[k] = np.exp(d * evals[k])
            k += 1
        else:
            expat, b = np.exp(d * evals[k]), evals[S + k]
            ec[k] = ec[k + 1] = expat * np.cos(d * b)
            es[k], es[k + 1] = expat * np.sin(d * b), -expat * np.sin(d * b)
            pt[k], pt[k + 1] = k + 1, k
            k += 2
    iexp = ec[:, None] * ievc + es[:, None] * ievc[pt]
    scale = np.abs(evec) @ (np.abs(ec)[:, None] * np.abs(ievc) + np.abs(es)[:, None] * np.abs(ievc[pt]))
    return np.abs(evec @ iexp), scale


CASES = [(S, C, kind) for S in (4, 3) for C in (1, 3, 4, 8, 32) for kind in ("real", "complex")]


@pytest.mark.parametrize("S,C,kind", CASES)
def test_matrices_match_restatement(S, C, kind):
    """Two eigen systems and two rate sets in one call (updateTransitionMatricesWithMultipleModels), every length of
    LENGTHS with every (system, rate set) pair, written to matrix buffers in reverse order."""
    first = _ComplexModel(S, 7 + S) if kind == "complex" else _real_model(S, 3)
    second = em.HKY(2.0, np.full(4, 0.25)) if S == 4 else _real_model(S, 5)
    flags = beagle.BeagleFlag.EIGEN_COMPLEX if kind == "complex" else 0
    systems = []
    for m in (first, second):
        e = m.getEigenDecomposition()
        # a complex instance takes real || imaginary parts: a real system has zero imaginary parts
        ev = np.concatenate([e.Eval, np.zeros(S)]) if flags and e.Eval.shape[0] == S else e.Eval
        systems.append((np.ascontiguousarray(e.Evec), np.ascontiguousarray(e.Ievc), np.ascontiguousarray(ev)))
    rng = np.random.default_rng(S * 100 + C)
    rates = [np.sort(rng.uniform(0.05, 3.0, C)), np.sort(rng.uniform(0.05, 3.0, C))]
    eig_idx, rate_idx, lens = np.meshgrid([0, 1], [0, 1], LENGTHS, indexing="ij")
    eig_idx, rate_idx, lens = (a.reshape(-1) for a in (eig_idx, rate_idx, lens))
    n = lens.shape[0]
    prob_idx = np.arange(n + 2)[::-1][:n].astype(np.int32)
    inst = GPU(3, 5, 3, S, 16, 2, n + 2, C, 0, [1, 0], 0, flags)
    try:
        for e, (evec, ievc, ev) in enumerate(systems):
            inst.setEigenDecomposition(e, evec, ievc, ev)
        for r in range(2):
            inst.setCategoryRatesWithIndex(r, rates[r])
        inst.updateTransitionMatricesWithMultipleModels(eig_idx.astype(np.int32), rate_idx.astype(np.int32), prob_idx,
                                                        None, None, lens.astype(np.float64), n)
        for q in range(n):
            got = np.zeros(C * S * S)
            inst.getTransitionMatrix(int(prob_idx[q]), got)
            got = got.reshape(C, S, S)
            evec, ievc, ev = systems[eig_idx[q]]
            for c in range(C):
                want, scale = _restated(evec, ievc, ev, lens[q] * rates[rate_idx[q]][c])
                assert np.all(np.abs(got[c] - want) <= 16 * EPS * scale + 1e-300), (q, c, got[c], want)
    finally:
        inst.finalize()


@pytest.mark.parametrize("S,C,kind", CASES)
def test_evaluation_matches_oracle(S, C, kind, monkeypatch):
    """One full evaluation per route against the oracle: the default walk (eigen form on a real system, matrix form on a
    complex one), the matrix-form walk, and the tensor walk (its Mpad / MTg copies; other C fall back to the FMA walk)."""
    tree, pats, model, site = H.synthetic_case(24, 200, categories=C, seed=20 + S + C, stateCount=S, rootHeight=0.5)
    if kind == "complex":
        model = _ComplexModel(S, 7 + S)
    o = tdl.BeagleDataLikelihoodDelegate(tree, pats, model, site, H.oracle_factory(report_flags=0),
                                         rescalingScheme=tdl.PartialsRescalingScheme.NONE)
    want = tdl.TreeDataLikelihood(o, tree).getLogLikelihood()
    for env in ({}, {"B200_EIGEN_WALK": "0"}, {"B200_WALK_VARIANT": "2"}):
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            d = tdl.BeagleDataLikelihoodDelegate(tree, pats, model, site, GPU, resourceList=[1, 0],
                                                 rescalingScheme=tdl.PartialsRescalingScheme.NONE)
            got = tdl.TreeDataLikelihood(d, tree).getLogLikelihood()
            d.finalize()
        assert np.isfinite(want) and abs(got - want) <= REL * abs(want), (env, got, want)
