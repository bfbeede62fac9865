"""Markov-jump counts and rewards on the device (b200SampleMarkovJumps, csrc/ancestral.cu).

The draws must be bit-identical to b200SampleAncestralStates.  The counts are checked against the numpy restatement
(oracle/markov_jumps.py) fed with the engine's own draws, eigen system, rates and lengths: every total within the sum of the
per-entry bounds of the values it adds.  Two checks do not depend on the formula: the prior identity with all tips gaps,
and the posterior expectation by exact enumeration with Van Loan conditional matrices."""
import ctypes as C
import itertools

import numpy as np
import pytest
from scipy.linalg import expm

from beast_mcmc_b200 import beagle
from harness import evomodel as em
from oracle import ancestral as anc
from oracle import markov_jumps as mj
from test_gpu_ancestral import BOUNDARY, NONE, Case, _shard_resource, _with_env

pytestmark = pytest.mark.gpu

OUT_OF_RANGE = beagle.BeagleErrorCode.OUT_OF_RANGE_ERROR
NO_IMPLEMENTATION = beagle.BeagleErrorCode.NO_IMPLEMENTATION_ERROR


def _registers(case, kind):
    Q = case.model.infinitesimalMatrix()
    S = case.S
    changes = Q - np.diag(np.diag(Q))
    if kind == "codon":                                 # synonymous and non-synonymous single-nucleotide changes
        syn = np.array([[em._AA[a] == em._AA[b] for b in em.SENSE_CODONS] for a in em.SENSE_CODONS])
        return np.stack([np.where(syn, changes, 0.0), np.where(~syn, changes, 0.0)])
    directed = np.zeros((S, S))
    directed[0, 1] = Q[0, 1]
    reward = np.diag((np.arange(S) == 1).astype(np.float64))
    return np.stack([changes, directed, reward])


def _row_lengths(case):
    return case.lengths[[r[0] for r in case.rows]]


def _jumps(case, inst, regs, seed=7, drawIndex=0, lengths=None, **kw):
    nb, pr, mi = case.arrays()
    lengths = _row_lengths(case) if lengths is None else lengths
    return inst.sampleMarkovJumps(nb, pr, mi, lengths, case.root, 0, 0, 0, 0, regs, seed, drawIndex, **kw)


def _weights(case, inst, seed=1):
    w = np.random.default_rng(seed).integers(1, 5, case.P).astype(np.float64)
    inst.setPatternWeights(w)
    return w


def _oracle(case, states, cats, regs, w, lengths=None):
    ed = case.model.getEigenDecomposition()
    lengths = _row_lengths(case) if lengths is None else lengths
    parents = [r[1] for r in case.rows]
    return mj.counts(parents, states, cats, lengths, case.rates, ed.Evec, ed.Ievc, ed.Eval, regs, w)


def _assert_counts(got, want, w, label):
    (_, _, branch, pattern), (_, obranch, opattern, bound) = got, want
    pb, bb = bound.sum(axis=1), bound @ w
    pr, br = np.abs(pattern - opattern) / pb, np.abs(branch - obranch)[:, 1:] / bb[:, 1:]
    print(f"{label}: worst pattern total {pr.max():.3e}, worst branch total {br.max():.3e} of the bound")
    assert (branch[:, 0] == 0).all()
    assert pr.max() <= 1.0 and br.max() <= 1.0, label


def _draws_and_counts(case, inst, kind, seed, drawIndex, label):
    regs = _registers(case, kind)
    w = _weights(case, inst)
    got = _jumps(case, inst, regs, seed, drawIndex)
    ref = case.sample(inst, seed, drawIndex)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), label
    _assert_counts(got, _oracle(case, got[0], got[1], regs, w), w, label)
    # one register alone: the same values as that register among several
    one = _jumps(case, inst, regs[:1], seed, drawIndex)
    assert np.array_equal(one[2], got[2][:1]) and np.array_equal(one[3], got[3][:1])
    return got


@pytest.mark.parametrize("S", [4, 20, 61])
@pytest.mark.parametrize("C", [1, 4])
def test_draws_unchanged_and_counts_match_oracle(S, C):
    T, P = (12, 300) if S == 4 else ((9, 160) if S == 20 else (7, 64))
    case = Case(S=S, C=C, T=T, P=P, seed=S + C)
    inst = case.create()
    case.evaluate(inst)
    _draws_and_counts(case, inst, "codon" if S == 61 else "nucleotide", 2024, 5, f"S={S} C={C}")
    if S == 61:
        _draws_and_counts(case, inst, "nucleotide", 2024, 6, f"S={S} C={C} changes/directed/reward")
    inst.finalize()


def test_single_precision_draws_unchanged_and_counts_match_oracle():
    case = Case(S=4, C=4, T=16, P=500, seed=41)
    inst = case.create(requirement=beagle.BeagleFlag.PRECISION_SINGLE)
    assert inst.getDetails().getFlags() & beagle.BeagleFlag.PRECISION_SINGLE
    case.evaluate(inst)
    _draws_and_counts(case, inst, "nucleotide", 11, 1, "single")
    inst.finalize()


def test_discrete_trait_shape():
    """S = 12, one category, one pattern, 200 tips: the warp kernel with a single pattern (phylogeography)"""
    case = Case(S=12, C=1, T=200, P=1, seed=12)
    inst = case.create()
    case.evaluate(inst)
    _draws_and_counts(case, inst, "nucleotide", 5, 0, "discrete trait")
    inst.finalize()


def test_prior_identity_all_gaps():
    """all tips gaps: every pattern is an independent draw from the prior, where E[register total] = t * pi^T M 1"""
    S, P = 4, 20_000
    case = Case(S=S, C=4, T=10, seed=30, partialTips=0, columns=np.full((10, P), S))
    inst = case.create()
    case.evaluate(inst)
    regs = _registers(case, "nucleotide")
    _, _, _, pattern = _jumps(case, inst, regs, 3, 0, states=False, categories=False, branchCounts=False)
    t = _row_lengths(case)[1:].sum() * float(case.weights @ case.rates)
    pi = case.model.getFrequencies()
    for g, want in ((0, t), (2, pi[1] * t)):                    # all changes (pi^T Q_offdiag 1 = 1), reward of state 1
        mean, se = pattern[g].mean(), pattern[g].std(ddof=1) / np.sqrt(P)
        print(f"register {g}: mean {mean:.6f}, want {want:.6f}, {abs(mean - want) / se:.2f} SE")
        assert abs(mean - want) <= 5 * se
    inst.finalize()


def test_posterior_expectation_by_enumeration():
    """4 tips, one column replicated: E[n | data] from the exact joint posterior with Van Loan conditional matrices"""
    S, P = 4, 20_000
    column = np.array([0, 1, 1, 3], dtype=np.int32)
    case = Case(S=S, C=2, T=4, seed=31, partialTips=0, columns=np.repeat(column[:, None], P, axis=1))
    inst = case.create()
    case.evaluate(inst)
    regs = _registers(case, "nucleotide")
    _, _, branch, pattern = _jumps(case, inst, regs, 8, 0, states=False, categories=False)
    Q = case.model.infinitesimalMatrix()
    lengths = _row_lengths(case)
    R = len(case.rows)
    parents = [r[1] for r in case.rows]
    mats = [None] + [np.stack([expm(Q * rc * lengths[r]) for rc in case.rates]) for r in range(1, R)]
    tipRows = {r: node for r, (node, _, _) in enumerate(case.rows) if node < case.T}
    tipL = {r: np.eye(S)[column[node]] for r, node in tipRows.items()}
    outcomes, probs = anc.enumerate_joint(parents, mats, tipL, case.weights, case.model.getFrequencies())
    internal = [r for r in range(R) if r not in tipL]
    for g in range(len(regs)):
        N = {(r, c): mj.van_loan(Q, regs[g], rc * lengths[r]) / mats[r][c] for r in range(1, R)
             for c, rc in enumerate(case.rates)}
        per = np.zeros((len(outcomes), R))
        for k, o in enumerate(outcomes):
            x = dict(zip(internal, o[1:]))
            x.update({r: column[node] for r, node in tipRows.items()})
            for r in range(1, R):
                per[k, r] = N[(r, o[0])][x[parents[r]], x[r]]
        want_pattern = probs @ per.sum(axis=1)
        mean, se = pattern[g].mean(), pattern[g].std(ddof=1) / np.sqrt(P)
        print(f"register {g}: mean {mean:.6f}, exact {want_pattern:.6f}, {abs(mean - want_pattern) / se:.2f} SE")
        assert abs(mean - want_pattern) <= 5 * se
        support = probs > 0
        for r in range(1, R):
            lo, hi = per[support, r].min(), per[support, r].max()
            want = probs @ per[:, r]
            assert abs(branch[g, r] / P - want) <= 5 * (hi - lo) / (2 * np.sqrt(P)) + 1e-12, (g, r)
    inst.finalize()


def test_repeated_calls_bit_identical_and_zero_lengths_give_zero():
    case = Case(S=4, C=4, T=20, P=300, seed=32)
    inst = case.create()
    case.evaluate(inst)
    _weights(case, inst)
    regs = _registers(case, "nucleotide")
    a, b = _jumps(case, inst, regs, 1, 0), _jumps(case, inst, regs, 1, 0)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    lengths = _row_lengths(case).copy()
    zero = np.arange(len(lengths)) % 3 == 1
    lengths[zero] = 0.0
    z = _jumps(case, inst, regs, 1, 0, lengths=lengths)
    assert np.array_equal(z[0], a[0]) and (z[2][:, zero] == 0).all()
    assert np.array_equal(z[2][:, ~zero], a[2][:, ~zero])
    allzero = _jumps(case, inst, regs, 1, 0, lengths=np.zeros(len(lengths)))
    assert (allzero[2] == 0).all() and (allzero[3] == 0).all()
    inst.finalize()


def test_virtual_cherries_on_off_bit_equal():
    case = Case(S=4, C=4, T=64, P=700, seed=13, partialTips=0)

    def run():
        inst = case.create()
        case.evaluate(inst)
        _weights(case, inst)
        out = _jumps(case, inst, _registers(case, "nucleotide"), 17, 9)
        inst.finalize()
        return out

    on = run()
    off = _with_env({"B200_VIRTUAL_CHERRIES": "0"}, run)
    assert all(np.array_equal(x, y) for x, y in zip(on, off))


def _move_branch_deferred(case, inst, lengths):
    node = case.ops[3][0]
    lengths[node] *= 1.7
    inst.updateTransitionMatrices(0, np.array([node], np.int32), None, None, lengths[[node]], 1)
    parent = {c: n for n, a, b in case.ops for c in (a, b)}
    by_node = {o[0]: o for o in case.ops}
    path, n = [], node
    while n != case.root:
        n = parent[n]
        path.append(by_node[n])
    flat = []
    for n, a, b in path:
        flat += [n, NONE, NONE, a, a, b, b]
    inst.updatePartials(np.array(flat, dtype=np.int32), len(path), NONE)


def test_pending_deferred_evaluation_is_flushed_first():
    case = Case(S=4, C=4, T=64, P=700, seed=14, partialTips=0)
    inst = case.create()
    case.evaluate(inst)
    out = np.zeros(1)
    inst.calculateRootLogLikelihoods(np.array([case.root], np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32),
                                     np.array([NONE], np.int32), 1, out)
    lengths = case.lengths.copy()
    _move_branch_deferred(case, inst, lengths)
    regs = _registers(case, "nucleotide")
    rowLengths = lengths[[r[0] for r in case.rows]]
    got = _jumps(case, inst, regs, 3, 4, lengths=rowLengths)
    fresh = case.create()
    case.evaluate(fresh, lengths)
    ref = _jumps(case, fresh, regs, 3, 4, lengths=rowLengths)
    margins = case.oracle_draws(inst, 3, 4)[2]
    ok = ~(margins < BOUNDARY).any(axis=0)
    assert ok.mean() >= 0.99
    assert np.array_equal(got[0][:, ok], ref[0][:, ok]) and np.array_equal(got[3][:, ok], ref[3][:, ok])
    inst.finalize(); fresh.finalize()


def test_rescaled_instance_counts_as_unscaled():
    case = Case(S=4, C=4, T=40, P=400, seed=12)
    regs = _registers(case, "nucleotide")
    plain = case.create()
    case.evaluate(plain)
    ref = _jumps(case, plain, regs, 5, 3)
    margins = case.oracle_draws(plain, 5, 3)[2]
    scaled = case.create(scaled=True)
    case.evaluate(scaled)
    got = _jumps(case, scaled, regs, 5, 3)
    ok = ~(margins < BOUNDARY).any(axis=0)
    assert np.array_equal(got[0][:, ok], ref[0][:, ok]) and np.array_equal(got[3][:, ok], ref[3][:, ok])
    plain.finalize(); scaled.finalize()


def _raw_call(lib, inst, case, regs, lengths, outs, nb=None, pr=None, mi=None, root=None, w=0, f=0, e=0, r=0, G=None,
              regsPtr=True, lengthsPtr=True):
    a_nb, a_pr, a_mi = case.arrays()
    ip = lambda a: np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int))
    dp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))
    ipo = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_int))
    nb = a_nb if nb is None else nb
    return lib.b200SampleMarkovJumps(inst.instance, ip(nb), ip(a_pr if pr is None else pr), ip(a_mi if mi is None else mi),
                                     dp(lengths) if lengthsPtr else None, len(nb), case.root if root is None else root,
                                     w, f, e, r, dp(regs) if regsPtr else None, len(regs) if G is None else G, 1, 0,
                                     ipo(outs[0]), ipo(outs[1]), dp(outs[2]), dp(outs[3]))


def _sentinel_outs(case, G):
    R = len(case.rows)
    return [np.full((R, case.P), -7, np.int32), np.full(case.P, -7, np.int32), np.full((G, R), -7.0),
            np.full((G, case.P), -7.0)]


def test_null_output_combinations_write_only_what_was_asked():
    case = Case(S=4, C=2, T=12, P=200, seed=33)
    inst = case.create()
    case.evaluate(inst)
    regs = np.ascontiguousarray(_registers(case, "nucleotide"))
    lengths = np.ascontiguousarray(_row_lengths(case))
    lib = beagle.load_library()
    full = _sentinel_outs(case, len(regs))
    assert _raw_call(lib, inst, case, regs, lengths, full) == 0
    for mask in itertools.product([False, True], repeat=4):
        outs = _sentinel_outs(case, len(regs))
        ask = [o if m else None for o, m in zip(outs, mask)]
        rc = _raw_call(lib, inst, case, regs, lengths, ask)
        if not (mask[2] or mask[3]):
            assert rc == OUT_OF_RANGE
            assert all((o == -7).all() for o in outs)
            continue
        assert rc == 0, mask
        for o, m, ref in zip(outs, mask, full):
            assert np.array_equal(o, ref) if m else (o == -7).all(), mask
    inst.finalize()


@pytest.mark.parametrize("S,P,g", [(4, 301, 3), (4, 2, 3), (20, 97, 2)])
def test_sharded_instance_matches_single_device(S, P, g):
    case = Case(S=S, C=2, T=10, P=P, seed=16 + P)
    res = _shard_resource(list(range(g)))
    whole, sharded = case.create(), case.create(resource=res)
    assert sharded.getDetails().getResourceNumber() == res
    regs = _registers(case, "nucleotide")
    w = np.random.default_rng(2).integers(1, 5, P).astype(np.float64)
    for inst in (whole, sharded):
        case.evaluate(inst)
        inst.setPatternWeights(w)
    a, b = _jumps(case, whole, regs, 21, 2), _jumps(case, sharded, regs, 21, 2)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[3], b[3])
    assert np.allclose(a[2], b[2], rtol=1e-12, atol=0)
    whole.finalize(); sharded.finalize()


def _create(case, eigenCount=1, requirement=0):
    inst = beagle.BeagleJNIImpl(case.T, case.N, case.T, case.S, case.P, eigenCount, case.N, case.C, 0, [1, 0], 0, requirement)
    inst.setStateFrequencies(0, case.model.getFrequencies())
    inst.setCategoryWeights(0, case.weights)
    inst.setCategoryRates(case.rates)
    for t in range(case.T):
        if t in case.tipPartials:
            inst.setTipPartials(t, case.tipPartials[t].ravel())
        else:
            inst.setTipStates(t, case.states[t])
    case.scaled = False
    return inst


def test_errors_return_their_code_and_launch_nothing():
    case = Case(S=4, C=4, T=20, P=300, seed=17, partialTips=0)
    inst = _create(case, eigenCount=2)
    ed = case.model.getEigenDecomposition()
    inst.setEigenDecomposition(0, ed.Evec.ravel(), ed.Ievc.ravel(), ed.Eval)
    lib = beagle.load_library()
    regs = np.ascontiguousarray(_registers(case, "nucleotide"))
    lengths = np.ascontiguousarray(_row_lengths(case))
    G = len(regs)
    R = len(case.rows)
    case.evaluate(inst)
    out = np.zeros(1)
    inst.calculateRootLogLikelihoods(np.array([case.root], np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32),
                                     np.array([NONE], np.int32), 1, out)
    before = _sentinel_outs(case, G)
    assert _raw_call(lib, inst, case, regs, lengths, before) == 0
    # deferred work pending: a refused call must leave it pending (nothing launched), the root call then fuses it
    node = case.ops[2][0]
    inst.updateTransitionMatrices(0, np.array([node], np.int32), None, None, case.lengths[[node]] * 1.3, 1)
    fused = lib.b200GetFusedLaunches(inst.instance)
    _, pr, _ = case.arrays()
    child = int(np.nonzero(pr > 0)[0][0])
    selfParent = pr.copy()
    selfParent[child] = child

    def lens(k, v):
        x = lengths.copy()
        x[k] = v
        return dict(lengths=x)

    bad = [dict(pr=selfParent), dict(root=-1), dict(w=10_000), dict(f=-1), dict(e=2), dict(e=-1), dict(e=1),   # slot 1 never set
           dict(r=10_000), dict(r=-1), dict(lengthsPtr=False), lens(3, -0.1), lens(R - 1, np.nan), lens(1, np.inf),
           dict(regsPtr=False), dict(G=0), dict(G=9), dict(noCounts=True)]
    for kw in bad:
        outs = _sentinel_outs(case, G)
        ask = list(outs)
        if kw.pop("noCounts", False):
            ask[2] = ask[3] = None
        L = kw.pop("lengths", lengths)
        assert _raw_call(lib, inst, case, regs, L, ask, **kw) == OUT_OF_RANGE, kw
        assert all((o == -7).all() for o in outs), kw
    by_node = {o[0]: o for o in case.ops}
    parent = {c: n for n, a, b in case.ops for c in (a, b)}
    path, n = [], node
    while n != case.root:
        n = parent[n]
        path.append(by_node[n])
    flat = []
    for n, a, b in path:
        flat += [n, NONE, NONE, a, a, b, b]
    inst.updatePartials(np.array(flat, dtype=np.int32), len(path), NONE)
    inst.calculateRootLogLikelihoods(np.array([case.root], np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32),
                                     np.array([NONE], np.int32), 1, out)
    assert lib.b200GetFusedLaunches(inst.instance) == fused + 1
    # back at the original lengths, a valid call gives what it gave before the refusals
    inst.updateTransitionMatrices(0, np.array([node], np.int32), None, None, case.lengths[[node]], 1)
    case.evaluate(inst)
    after = _sentinel_outs(case, G)
    assert _raw_call(lib, inst, case, regs, lengths, after) == 0
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    # row 0's length is not read
    assert _raw_call(lib, inst, case, regs, lens(0, np.nan)["lengths"], after) == 0
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    inst.finalize()


def test_complex_eigen_system_and_large_state_count_are_not_implemented():
    case = Case(S=4, C=1, T=6, P=50, seed=18, partialTips=0)
    inst = _create(case, requirement=beagle.BeagleFlag.EIGEN_COMPLEX)
    ed = case.model.getEigenDecomposition()
    inst.setEigenDecomposition(0, ed.Evec.ravel(), ed.Ievc.ravel(), np.concatenate([ed.Eval, [0.0, 0.3, -0.3, 0.0]]))
    case.evaluate(inst)
    lib = beagle.load_library()
    regs = np.ascontiguousarray(_registers(case, "nucleotide"))
    outs = _sentinel_outs(case, len(regs))
    assert _raw_call(lib, inst, case, regs, np.ascontiguousarray(_row_lengths(case)), outs) == NO_IMPLEMENTATION
    assert all((o == -7).all() for o in outs)
    # a real system in the same complex-capable instance is served
    inst.setEigenDecomposition(0, ed.Evec.ravel(), ed.Ievc.ravel(), np.concatenate([ed.Eval, np.zeros(4)]))
    assert _raw_call(lib, inst, case, regs, np.ascontiguousarray(_row_lengths(case)), outs) == 0
    inst.finalize()
    big = Case(S=200, C=1, T=3, P=4, seed=19, partialTips=0)
    inst = big.create()
    big.evaluate(inst)
    regs = np.ascontiguousarray(np.eye(200)[None])
    outs = _sentinel_outs(big, 1)
    assert _raw_call(lib, inst, big, regs, np.ascontiguousarray(_row_lengths(big)), outs) == NO_IMPLEMENTATION
    assert all((o == -7).all() for o in outs)
    inst.finalize()
