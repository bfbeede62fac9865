"""Markov-jump counts and rewards conditioned on sampled ancestral states, restated in numpy (the checker of
b200SampleMarkovJumps, csrc/ancestral.cu; Minin & Suchard 2008, BEAST's MarkovJumpsCore).

With the real eigen system Q = V diag(lam) V^-1 and a register matrix M_g (counts: M_ij = Q_ij R_ij off the diagonal, zero
diagonal; rewards: M = diag(r)), for the branch above row r >= 1 in category c, tau = r_c * edgeLengths[r]:
  I_kl(tau) = tau * exp(lam_l tau) * phi((lam_k - lam_l) tau),  phi(x) = expm1(x) / x,  phi(0) = 1
              (evaluated with the larger of lam_k, lam_l in the exponential: the same value, and expm1 cannot overflow)
  W_g = V^-1 M_g V,  E = V (W_g o I(tau)) V^-1,  Phat = |V diag(exp(lam tau)) V^-1| (entrywise)
  N[i][j] = E[i][j] / Phat[i][j], and 0 where Phat[i][j] = 0
Per pattern p with drawn category c and states x: n_g[r][p] = N_g,c,r[x_parent(r)][x_r] (row 0 contributes nothing);
branch totals sum_p w_p n_g[r][p] (w the pattern weights), pattern totals sum_{r >= 1} n_g[r][p].

``van_loan`` is the exact joint matrix through a matrix exponential, independent of the eigen form.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import expm


def phi(x):
    """expm1(x) / x, 1 at x = 0"""
    x = np.asarray(x, dtype=np.float64)
    out = np.ones_like(x)
    nz = x != 0.0
    out[nz] = np.expm1(x[nz]) / x[nz]
    return out


def integral(lam, tau):
    """I_kl(tau) = int_0^tau exp(lam_k s + lam_l (tau - s)) ds"""
    lk, ll = lam[:, None], lam[None, :]
    e = np.exp(tau * lam)
    emax = np.where(lk >= ll, e[:, None], e[None, :])
    return tau * emax * phi(-np.abs(lk - ll) * tau)


def transition(V, Vi, lam, tau):
    """Phat: |V diag(exp(lam tau)) V^-1| entrywise"""
    return np.abs((V * np.exp(tau * lam)[None, :]) @ Vi)


def joint(V, Vi, lam, M, tau):
    """E = V (W o I(tau)) V^-1, W = V^-1 M V: the expected register total along the branch jointly with its end state"""
    return V @ ((Vi @ M @ V) * integral(lam, tau)) @ Vi


def conditional(V, Vi, lam, M, tau):
    """(N, Phat): the expectation conditioned on both end states"""
    E, P = joint(V, Vi, lam, M, tau), transition(V, Vi, lam, tau)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(P > 0.0, E / np.where(P > 0.0, P, 1.0), 0.0), P


def van_loan(Q, M, tau):
    """the top-right block of expm([[Q tau, M tau], [0, Q tau]]): the exact joint matrix (Van Loan 1978)"""
    S = Q.shape[0]
    A = np.zeros((2 * S, 2 * S))
    A[:S, :S] = Q * tau
    A[:S, S:] = M * tau
    A[S:, S:] = Q * tau
    return expm(A)[:S, S:]


def entry_bound(want, got, Phat, Pexact):
    """the per-entry tolerance of a conditional value: 1e-11 |want| + 1e-14 (1 + |got|) / min(Phat, Pexact)"""
    with np.errstate(divide="ignore"):
        return 1e-11 * np.abs(want) + 1e-14 * (1.0 + np.abs(got)) / np.minimum(Phat, Pexact)


def counts(parentRows, states, categories, lengths, rates, V, Vi, lam, registers, patternWeights):
    """parentRows [rows] (row 0 the root), states int [rows][P], categories int [P], lengths [rows], rates [C],
    the eigen system (V, V^-1, lam), registers [G][S][S], patternWeights [P].
    Returns (n [G][rows][P], branch totals [G][rows], pattern totals [G][P], bound [G][rows][P]) where bound is entry_bound
    of each looked-up value against the exact conditional (scipy expm of Q tau) with got = want."""
    V, Vi, lam = (np.asarray(a, dtype=np.float64) for a in (V, Vi, lam))
    registers = np.asarray(registers, dtype=np.float64).reshape(-1, lam.size, lam.size)
    states, categories = np.asarray(states), np.asarray(categories)
    G, R, P = registers.shape[0], len(parentRows), states.shape[1]
    Q = (V * lam[None, :]) @ Vi
    n = np.zeros((G, R, P))
    bound = np.zeros((G, R, P))
    cols = np.arange(P)
    for r in range(1, R):
        i, j = states[parentRows[r]], states[r]
        for c in np.unique(categories):
            sel = cols[categories == c]
            tau = rates[c] * lengths[r]
            Pexact = expm(Q * tau)
            for g in range(G):
                N, Phat = conditional(V, Vi, lam, registers[g], tau)
                v = N[i[sel], j[sel]]
                n[g, r, sel] = v
                bound[g, r, sel] = entry_bound(v, v, Phat[i[sel], j[sel]], Pexact[i[sel], j[sel]])
    pattern = np.zeros((G, P))
    for r in range(1, R):                                  # in row order, as the kernels add
        pattern += n[:, r, :]
    branch = n @ np.asarray(patternWeights, dtype=np.float64)
    return n, branch, pattern, bound
