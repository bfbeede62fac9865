"""Complete substitution histories by uniformization, restated in numpy (the checker of b200SampleSubstitutionHistories,
csrc/ancestral.cu; DESIGN.md section 7.3).

With the generator Q, mu = max_i -Q_ii and R = I + Q/mu (R = I when mu = 0), for the branch above row r >= 1 in the drawn
category c, tau = r_c * lengths[r], parent state a and own state b:
  1. n, the number of uniformized jumps, is drawn with weights pi_n (R^n)[a][b], n = 0..N, pi_0 = exp(-mu tau),
     pi_n = pi_{n-1} mu tau / n, N = ceil(mu tau_max + 12 sqrt(mu tau_max) + 12) (tau_max over rows >= 1 and all categories)
  2. s_k, k = 1..n-1, with weights R[s_{k-1}][j] (R^{n-k})[j][b] over j (s_0 = a, s_n = b)
  3. U_0 = 0, U_k = 1 - (1 - U_{k-1}) v_k^{1/(n-k+1)}, evaluated as U_{k-1} - (1 - U_{k-1}) expm1(log(v_k) / (n-k+1))
  4. a jump with s_k = s_{k-1} is virtual; every other is an event (time lengths[r] U_k, new state s_k)
Each draw is oracle.ancestral.draw (the sampler's inverse CDF); when every weight of the n draw is 0, n = 0.  Uniform j of a
(row, pattern) pair is word j mod 4 of the Philox4x64-10 block at counter (drawIndex, global pattern, row, 1 + j // 4):
j = 0 draws n, j = 1..n-1 the states, j = n..2n-1 are the v_k.
Registers: n_g = sum over events (i -> j) of M_g[i][j] / Q[i][j] + sum over segments of M_g[s][s] tau (U_{k+1} - U_k), in the
order the kernel adds them: for k = 1..n the sojourn before jump k, then the jump; the last segment (U_{n+1} = 1) at the end.
"""
from __future__ import annotations

import math

import numpy as np

from oracle.ancestral import draw

_M32 = np.uint64(0xFFFFFFFF)
_MUL = (np.uint64(0xD2E7470EE14C6C93), np.uint64(0xCA5A826395121157))
_WEYL = (np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBB67AE8584CAA73B))


def _mulhilo(a, b):
    """(high, low) 64-bit words of the 128-bit product of uint64 arrays a and b"""
    a_lo, a_hi = a & _M32, a >> np.uint64(32)
    b_lo, b_hi = b & _M32, b >> np.uint64(32)
    ll, hl, lh, hh = a_lo * b_lo, a_hi * b_lo, a_lo * b_hi, a_hi * b_hi
    cross = (ll >> np.uint64(32)) + (hl & _M32) + lh
    return hh + (hl >> np.uint64(32)) + (cross >> np.uint64(32)), a * b


def philox_words(seed, c0, c1, c2, c3):
    """All four words of the Philox4x64-10 block at counter (c0, c1, c2, c3) under key (seed, 0), vectorized over the
    counters: uint64 [..., 4]."""
    with np.errstate(over="ignore"):
        c = [np.atleast_1d(np.asarray(x, dtype=np.uint64)) for x in np.broadcast_arrays(c0, c1, c2, c3)]
        k0, k1 = np.uint64(seed), np.uint64(0)
        for r in range(10):
            if r > 0:
                k0, k1 = k0 + _WEYL[0], k1 + _WEYL[1]
            hi0, lo0 = _mulhilo(c[0], _MUL[0])
            hi1, lo1 = _mulhilo(c[2], _MUL[1])
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, axis=-1)


def uniforms(seed, drawIndex, patterns, row, count):
    """[len(patterns)][count]: uniforms j = 0..count-1 of the pairs (row, pattern) for each global pattern index"""
    patterns = np.atleast_1d(np.asarray(patterns, dtype=np.uint64))
    blocks = (count + 3) // 4
    w = philox_words(seed, drawIndex, patterns[:, None], row, 1 + np.arange(blocks, dtype=np.uint64)[None, :])
    x = w.reshape(len(patterns), 4 * blocks)[:, :count]
    return (x >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def uniformized(Q):
    """(mu, R) of a generator"""
    Q = np.asarray(Q, dtype=np.float64)
    S = Q.shape[0]
    mu = float(max(0.0, np.max(-np.diag(Q))))
    R = np.eye(S) + Q / mu if mu > 0.0 else np.eye(S)
    return mu, R


def truncation(x_max):
    """N for mu tau_max = x_max"""
    return int(math.ceil(x_max + 12.0 * math.sqrt(x_max) + 12.0))


def powers(R, N):
    """[N + 1][S][S]: R^n by v_n = R v_{n-1} for every column at once"""
    out = np.empty((N + 1,) + R.shape)
    out[0] = np.eye(R.shape[0])
    for n in range(1, N + 1):
        out[n] = R @ out[n - 1]
    return out


def poisson_weights(x, N):
    """pi_n, n = 0..N, in the kernel's recurrence"""
    pi = np.empty(N + 1)
    p = math.exp(-x)
    for n in range(N + 1):
        pi[n] = p
        p = p * x / (n + 1)
    return pi


def history(a, b, tau, mu, R, Rn, u):
    """One history of a branch: (n, U [n], s [n + 1] with s[0] = a, smallest draw margin).  Rn = powers(R, N), u the pair's
    uniforms (at least 2N of them)."""
    N = Rn.shape[0] - 1
    pi = poisson_weights(mu * tau, N)
    w = pi * Rn[:, a, b]
    if w.any():
        n, margin = draw(w, u[0])
    else:
        n, margin = 0, np.inf
    s = [a]
    for k in range(1, n):
        wk = R[s[-1]] * Rn[n - k][:, b]
        j, m = draw(wk, u[k])
        margin = min(margin, m)
        s.append(j)
    if n > 0:
        s.append(b)
    U, prev = [], 0.0
    with np.errstate(divide="ignore"):
        for k in range(1, n + 1):
            prev = prev - (1.0 - prev) * np.expm1(np.log(u[n + k - 1]) / (n - k + 1))
            U.append(float(prev))
    return n, np.asarray(U), np.asarray(s), margin


def registers_of(U, s, tau, Q, M):
    """n_g of one history for registers M [G][S][S], in the kernel's order of addition"""
    reg = np.zeros(M.shape[0])
    prev = 0.0
    for k in range(1, len(U) + 1):
        i, j = s[k - 1], s[k]
        reg += M[:, i, i] * tau * (U[k - 1] - prev)
        if j != i:
            reg += M[:, i, j] / Q[i, j]
        prev = U[k - 1]
    return reg + M[:, s[-1], s[-1]] * tau * (1.0 - prev)


def events_of(U, s, length):
    """(times, new states) of the non-virtual jumps"""
    real = s[1:] != s[:-1]
    return length * U[real], s[1:][real]


def histories(parentRows, states, categories, lengths, rates, Q, registers, patternWeights, seed, drawIndex,
              patternOffset=0):
    """parentRows [rows] (row 0 the root), states int [rows][P], categories int [P], lengths [rows], rates [C], Q [S][S],
    registers [G][S][S], patternWeights [P].  Returns a dict: perRow [G][rows][P], branch [G][rows], pattern [G][P],
    jumps int [rows][P], times and eventStates (in (row, pattern, time) order), margins [rows][P] (the smallest CDF margin
    of each pair's draws, inf for row 0), N."""
    Q = np.asarray(Q, dtype=np.float64)
    registers = np.asarray(registers, dtype=np.float64).reshape(-1, Q.shape[0], Q.shape[0])
    states, categories = np.asarray(states), np.asarray(categories)
    rates, lengths = np.asarray(rates, dtype=np.float64), np.asarray(lengths, dtype=np.float64)
    G, R, P = registers.shape[0], len(parentRows), states.shape[1]
    mu, Rm = uniformized(Q)
    tau_max = max([float(np.max(lengths[r] * rates)) for r in range(1, R)] + [0.0])
    N = truncation(mu * tau_max)
    Rn = powers(Rm, N)
    perRow = np.zeros((G, R, P))
    jumps = np.zeros((R, P), dtype=np.int32)
    margins = np.full((R, P), np.inf)
    times, evStates = [], []
    for r in range(1, R):
        u_all = uniforms(seed, drawIndex, patternOffset + np.arange(P), r, max(2 * N, 1))
        for p in range(P):
            a, b = int(states[parentRows[r], p]), int(states[r, p])
            tau = lengths[r] * rates[categories[p]]
            n, U, s, margins[r, p] = history(a, b, tau, mu, Rm, Rn, u_all[p])
            perRow[:, r, p] = registers_of(U, s, tau, Q, registers)
            t, e = events_of(U, s, lengths[r])
            jumps[r, p] = len(t)
            times.append(t)
            evStates.append(e)
    pattern = np.zeros((G, P))
    for r in range(1, R):                                  # in row order, as the kernel adds
        pattern += perRow[:, r, :]
    return dict(perRow=perRow, branch=perRow @ np.asarray(patternWeights, dtype=np.float64), pattern=pattern, jumps=jumps,
                times=np.concatenate(times) if times else np.zeros(0),
                eventStates=np.concatenate(evStates).astype(np.int32) if evStates else np.zeros(0, np.int32),
                margins=margins, N=N)
