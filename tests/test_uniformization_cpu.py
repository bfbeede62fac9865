"""The uniformization restatement (oracle/uniformization.py) against results that do not depend on it: the matrix
exponential, Van Loan's conditional expectations, the no-event probability, and numpy's own Philox generator."""
import numpy as np
import pytest
from scipy.linalg import expm

import helpers as H  # noqa: F401  (sets sys.path)
from harness import evomodel as em
from oracle import ancestral as anc
from oracle import markov_jumps as mj
from oracle import uniformization as un


def _jc69():
    return (np.ones((4, 4)) - 4 * np.eye(4)) / 3


def _gtr():
    return em.GTR(1.0, 4.0, 0.7, 1.2, 5.0, 1.0, np.array([0.30, 0.22, 0.24, 0.24])).infinitesimalMatrix()


def _generator(off):
    return off - np.diag(off.sum(axis=1))


def _cyclic():
    """4-state non-reversible: a strong cycle 0 -> 1 -> 2 -> 3 -> 0 gives a complex pair"""
    off = np.full((4, 4), 0.05) - 0.05 * np.eye(4)
    for i in range(4):
        off[i, (i + 1) % 4] = 1.5
    return _generator(off)


def _asymmetric12():
    """12-state asymmetric location model (discrete phylogeography), some rates zero"""
    rng = np.random.default_rng(12)
    off = rng.uniform(0.0, 1.0, (12, 12)) * (rng.random((12, 12)) < 0.6)
    np.fill_diagonal(off, 0.0)
    return _generator(off)


MODELS = {"jc69": _jc69, "gtr": _gtr, "cyclic": _cyclic, "asym12": _asymmetric12}


def test_models_cover_complex_eigenvalues():
    for name in ("cyclic", "asym12"):
        assert np.abs(np.linalg.eigvals(MODELS[name]()).imag).max() > 1e-3, name


@pytest.mark.parametrize("name", sorted(MODELS))
def test_truncated_series_equals_matrix_exponential(name):
    Q = MODELS[name]()
    mu, R = un.uniformized(Q)
    for x in (1e-4, 0.3, 3.0, 40.0, 250.0, 700.0):             # mu tau up to the cap
        tau = x / mu
        N = un.truncation(x)
        series = np.einsum("n,nij->ij", un.poisson_weights(x, N), un.powers(R, N))
        err = np.abs(series - expm(Q * tau)).max()
        assert err <= 1e-13, (name, x, err)


def _draws(Q, a, b, tau, count, seed=5):
    """count histories of one (a, b, tau), one per pattern of row 1"""
    mu, R = un.uniformized(Q)
    N = un.truncation(mu * tau)
    Rn = un.powers(R, N)
    u = un.uniforms(seed, 0, np.arange(count), 1, 2 * N)
    return [un.history(a, b, tau, mu, R, Rn, u[p]) for p in range(count)]


def _registers(Q):
    S = Q.shape[0]
    changes = Q - np.diag(np.diag(Q))
    directed = np.zeros((S, S))
    i, j = np.argwhere(changes > 0)[0]
    directed[i, j] = Q[i, j]
    reward = np.diag((np.arange(S) == 1).astype(np.float64))
    mixed = 0.5 * changes + np.diag(np.linspace(0.0, 1.0, S))
    return np.stack([changes, directed, reward, mixed])


CASES = [("jc69", 0, 2, 0.4), ("jc69", 1, 1, 1.2), ("gtr", 0, 2, 0.3), ("gtr", 3, 3, 0.8), ("cyclic", 0, 3, 0.7),
         ("cyclic", 2, 2, 1.5), ("asym12", 0, 5, 0.6), ("asym12", 4, 4, 0.9)]


@pytest.mark.parametrize("name,a,b,tau", CASES)
def test_sampled_totals_match_van_loan(name, a, b, tau):
    Q = MODELS[name]()
    M = _registers(Q)
    count = 20_000
    hist = _draws(Q, a, b, tau, count)
    vals = np.array([un.registers_of(U, s, tau, Q, M) for _, U, s, _ in hist])
    assert all(s[0] == a and s[-1] == b for _, _, s, _ in hist)
    P = expm(Q * tau)[a, b]
    for g in range(len(M)):
        want = mj.van_loan(Q, M[g], tau)[a, b] / P
        mean, se = vals[:, g].mean(), vals[:, g].std(ddof=1) / np.sqrt(count)
        print(f"{name} {a}->{b} tau {tau} register {g}: mean {mean:.6f}, Van Loan {want:.6f}, "
              f"{abs(mean - want) / max(se, 1e-300):.2f} SE")
        assert abs(mean - want) <= 5 * se + 1e-12, (name, g)


@pytest.mark.parametrize("name,a,tau", [("jc69", 1, 1.2), ("gtr", 3, 0.8), ("cyclic", 2, 1.5), ("asym12", 4, 0.9)])
def test_no_event_probability(name, a, tau):
    Q = MODELS[name]()
    count = 20_000
    hist = _draws(Q, a, a, tau, count, seed=6)
    none = np.array([len(un.events_of(U, s, 1.0)[0]) == 0 for _, U, s, _ in hist])
    want = np.exp(Q[a, a] * tau) / expm(Q * tau)[a, a]
    se = np.sqrt(want * (1 - want) / count)
    print(f"{name}: P(no event) {none.mean():.5f}, want {want:.5f}")
    assert abs(none.mean() - want) <= 5 * se


def test_jump_times_ascend_within_the_branch():
    Q = _asymmetric12()
    for n, U, s, _ in _draws(Q, 0, 5, 2.0, 2000):
        assert len(U) == n and len(s) == n + 1
        assert np.all(np.diff(U) >= 0) and (n == 0 or (0 <= U[0] and U[-1] <= 1))


@pytest.mark.parametrize("counter", [(5, 3, 7, 1), (0, 0, 0, 0), (2 ** 64 - 1, 12345, 2 ** 40, 99), (9, 2 ** 63, 1, 2)])
def test_philox_words_equal_numpy(counter):
    seed = 2024
    c0, c1, c2, c3 = counter
    ctr = (c0 + c1 * 2 ** 64 + c2 * 2 ** 128 + c3 * 2 ** 192 - 1) % 2 ** 256    # numpy advances before a block
    want = np.random.Philox(key=seed, counter=ctr).random_raw(4)
    assert np.array_equal(un.philox_words(seed, *counter)[0], want)


def test_uniform_stream_layout():
    """uniform j is word j mod 4 of block 1 + j // 4; block 0 word 0 is the sampler's uniform"""
    u = un.uniforms(11, 3, [0, 17], 4, 10)
    for p, pat in enumerate((0, 17)):
        for j in range(10):
            x = un.philox_words(11, 3, pat, 4, 1 + j // 4)[0, j % 4]
            assert u[p, j] == (int(x) >> 11) * 2.0 ** -53
        w0 = un.philox_words(11, 3, pat, 4, 0)[0, 0]
        assert anc.uniform(11, 3, pat, 4) == (int(w0) >> 11) * 2.0 ** -53
