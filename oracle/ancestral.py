"""Joint ancestral-state sampling restated in numpy (the checker of b200SampleAncestralStates, csrc/ancestral.cu).

Per pattern p, with the rows in pre-order (row 0 the root):
  root : (c, i) drawn with probability proportional to w_c * pi_i * Lroot_c[p][i], items category-major
  row r: j given the parent row's state i and the root's category c, proportional to P_c[i][j] * L_r,c[p][j]; a compact tip
         keeps its observed state, a gap / unknown state (>= S) draws proportional to P_c[i][j]
Each draw is an inverse CDF in item order with sequential fp64 cumulative sums: the first item whose cumulative sum exceeds
u * total, else the last item of positive weight, else item 0.  u = (x >> 11) * 2^-53 with x the first output word of
Philox4x64-10 -- numpy.random.Philox itself -- under key seed and counter (drawIndex, global pattern, row, 0).

``enumerate_joint`` is the exact distribution of one pattern's (category, internal states) by enumeration, for tiny trees.
"""
from __future__ import annotations

import itertools

import numpy as np

_TWO64 = 1 << 64
_TWO256 = 1 << 256


def uniform(seed: int, drawIndex: int, pattern: int, row: int) -> float:
    """The uniform of one draw.  numpy's Philox advances its counter by one BEFORE it produces a block, so the block at
    counter n is the first output of a generator started at n - 1 (words little-endian: word 0 = drawIndex)."""
    ctr = (drawIndex + pattern * _TWO64 + row * _TWO64 * _TWO64 - 1) % _TWO256
    x = int(np.random.Philox(key=seed, counter=ctr).random_raw())
    return (x >> 11) * 2.0 ** -53


def draw(weights: np.ndarray, u: float):
    """(item, margin): the inverse-CDF pick and the distance of u from the nearest CDF boundary (in units of u)."""
    cum = np.cumsum(weights)                    # sequential fp64 sums, as the kernels add
    total = cum[-1]
    t = u * total
    hit = np.nonzero(t < cum)[0]
    if hit.size:
        j = int(hit[0])
    else:
        pos = np.nonzero(weights > 0.0)[0]
        j = int(pos[-1]) if pos.size else 0
    margin = float(np.min(np.abs(t - cum)) / total) if total > 0.0 and np.isfinite(total) else np.inf
    return j, margin


def sample(rows, rootBuffer, partials, tipStates, matrices, weights, freqs, seed, drawIndex, patternOffset=0):
    """rows: [(node buffer, parent row, matrix index)] in pre-order (row 0's buffer and matrix are not read);
    partials: buffer -> [C][P][S] (the root and every row given as partials); tipStates: buffer -> [P] compact states;
    matrices: matrix index -> [C][S][S] (P_c[i][j]); weights [C], freqs [S].
    Returns (states int32 [rows][P], categories int32 [P], margins [rows][P])."""
    weights = np.asarray(weights, dtype=np.float64)
    freqs = np.asarray(freqs, dtype=np.float64)
    root = partials[rootBuffer]
    C, P, S = root.shape
    count = len(rows)
    states = np.zeros((count, P), dtype=np.int32)
    cats = np.zeros(P, dtype=np.int32)
    margins = np.full((count, P), np.inf)
    wf = weights[:, None] * freqs[None, :]
    for p in range(P):
        q, margins[0, p] = draw((wf * root[:, p, :]).reshape(-1), uniform(seed, drawIndex, patternOffset + p, 0))
        c = q // S
        cats[p], states[0, p] = c, q % S
        for r in range(1, count):
            buf, parent, mat = rows[r]
            i = states[parent, p]
            row = matrices[mat][c, i, :]
            if buf in tipStates:
                s = int(tipStates[buf][p])
                if 0 <= s < S:
                    states[r, p] = s
                    continue
                w = row.copy()
            else:
                w = row * partials[buf][c, p, :]
            states[r, p], margins[r, p] = draw(w, uniform(seed, drawIndex, patternOffset + p, r))
    return states, cats, margins


def enumerate_joint(parents, matrices_of_rows, tipL, weights, freqs):
    """Exact joint posterior of ONE pattern over (category, states of the rows not in tipL).

    parents[r]: parent row (parents[0] = -1); matrices_of_rows[r]: [C][S][S] of the branch above row r; tipL: row -> [S]
    likelihood of a tip row (indicator of its state, all ones for a gap, or its partials), summed out through its branch.
    Returns (outcomes [(c, state of each internal row in row order)], probabilities)."""
    weights = np.asarray(weights, dtype=np.float64)
    freqs = np.asarray(freqs, dtype=np.float64)
    S = freqs.size
    internal = [r for r in range(len(parents)) if r not in tipL]
    outcomes, probs = [], []
    for c in range(weights.size):
        for xs in itertools.product(range(S), repeat=len(internal)):
            x = dict(zip(internal, xs))
            pr = weights[c] * freqs[x[0]]
            for r in range(1, len(parents)):
                M = matrices_of_rows[r][c]
                i = x[parents[r]]
                pr *= M[i] @ tipL[r] if r in tipL else M[i, x[r]]
            outcomes.append((c,) + xs)
            probs.append(pr)
    probs = np.asarray(probs)
    return outcomes, probs / probs.sum()
