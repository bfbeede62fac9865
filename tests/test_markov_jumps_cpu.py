"""The Markov-jump restatement (oracle/markov_jumps.py) against the exact joint matrix of Van Loan's block exponential, on
models with degenerate (JC69), distinct (GTR), random (20 states) and codon (MG94, 61 states) spectra.  CPU only."""
import numpy as np
import pytest

from harness import evomodel as em
from oracle import markov_jumps as mj

TAUS = np.geomspace(1e-4, 10.0, 40)


def _models():
    rng = np.random.default_rng(20)
    return {
        "JC69": em.SubstitutionModel(np.ones(6), np.full(4, 0.25)),
        "GTR": em.GTR(1.0, 4.0, 0.7, 1.2, 5.0, 1.0, np.array([0.30, 0.22, 0.24, 0.24])),
        "random20": em.SubstitutionModel(rng.uniform(0.2, 3.0, 190), rng.dirichlet(np.full(20, 5.0))),
        "MG94": em.MG94HKYCodonModel(1.0, 0.3, 2.0),
    }


def _registers(Q):
    """all changes, one directed transition, a reward indicator of state 1"""
    S = Q.shape[0]
    changes = Q - np.diag(np.diag(Q))
    one = np.zeros((S, S))
    one[0, 1] = Q[0, 1] if Q[0, 1] > 0 else changes[0].max()
    reward = np.zeros((S, S))
    reward[1, 1] = 1.0
    return {"changes": changes, "directed": one, "reward": reward}


@pytest.mark.parametrize("name", ["JC69", "GTR", "random20", "MG94"])
def test_eigen_formula_matches_van_loan(name):
    model = _models()[name]
    ed = model.getEigenDecomposition()
    V, Vi, lam = ed.Evec, ed.Ievc, ed.Eval
    Q = model.infinitesimalMatrix()
    worst_joint = worst_cond = 0.0
    for rname, M in _registers(Q).items():
        for tau in TAUS:
            E = mj.joint(V, Vi, lam, M, tau)
            want = mj.van_loan(Q, M, tau)
            worst_joint = max(worst_joint, np.max(np.abs(E - want)) / (1e-14 * max(1.0, tau)))
            got, Phat = mj.conditional(V, Vi, lam, M, tau)
            Pexact = mj.expm(Q * tau)
            pos = (Phat > 0) & (Pexact > 0)
            wantN = want[pos] / Pexact[pos]
            bound = mj.entry_bound(wantN, got[pos], Phat[pos], Pexact[pos])
            worst_cond = max(worst_cond, np.max(np.abs(got[pos] - wantN) / bound))
    print(f"{name}: worst joint error {worst_joint:.3f}, worst conditional error {worst_cond:.3f} of the bound")
    assert worst_joint <= 1.0 and worst_cond <= 1.0


def test_phi_at_zero_and_tiny_arguments():
    assert mj.phi(np.array([0.0]))[0] == 1.0
    for x in (1e-300, -1e-300, 1e-20, -1e-12, 1e-8, -1e-5):
        series = 1.0 + x / 2 + x * x / 6 + x ** 3 / 24
        assert abs(mj.phi(np.array([x]))[0] - series) <= 4e-16, x
    assert np.isfinite(mj.integral(np.array([0.0, -800.0]), 10.0)).all()        # no expm1 overflow


@pytest.mark.parametrize("name", ["JC69", "GTR", "random20", "MG94"])
def test_stationary_identity(name):
    """pi^T E 1 = tau pi^T M 1: at stationarity the expected register total is tau times its rate"""
    model = _models()[name]
    ed = model.getEigenDecomposition()
    pi, Q = model.getFrequencies(), model.infinitesimalMatrix()
    for M in _registers(Q).values():
        for tau in (1e-3, 0.1, 1.0, 7.0):
            lhs = pi @ mj.joint(ed.Evec, ed.Ievc, ed.Eval, M, tau) @ np.ones(pi.size)
            rhs = tau * (pi @ M @ np.ones(pi.size))
            assert abs(lhs - rhs) <= 1e-12 * max(1.0, abs(rhs)), (tau, lhs, rhs)


def test_counts_looks_up_the_drawn_pairs():
    """counts() against a direct per-pattern lookup on a 3-row tree with two categories"""
    model = _models()["GTR"]
    ed = model.getEigenDecomposition()
    Q = model.infinitesimalMatrix()
    regs = np.stack(list(_registers(Q).values()))
    parents = [-1, 0, 0]
    states = np.array([[0, 1, 2, 3, 0], [1, 1, 0, 3, 2], [0, 2, 2, 1, 3]])
    cats = np.array([0, 1, 1, 0, 1])
    lengths, rates, w = np.array([9.9, 0.1, 0.0]), np.array([0.5, 1.5]), np.array([1.0, 2.0, 1.0, 3.0, 1.0])
    n, branch, pattern, bound = mj.counts(parents, states, cats, lengths, rates, ed.Evec, ed.Ievc, ed.Eval, regs, w)
    for g in range(regs.shape[0]):
        for p in range(5):
            N = mj.conditional(ed.Evec, ed.Ievc, ed.Eval, regs[g], rates[cats[p]] * 0.1)[0]
            assert n[g, 1, p] == N[states[0, p], states[1, p]]
    assert (n[:, 0] == 0).all() and (n[:, 2] == 0).all()                    # root row and a zero-length branch
    assert np.allclose(branch, n @ w) and np.allclose(pattern, n.sum(axis=1))
    assert (bound[:, 1] > 0).all() and np.isfinite(bound[:, 1]).all()
