"""Complete substitution histories by uniformization on the device (b200SampleSubstitutionHistories, csrc/ancestral.cu).

The end states must be bit-identical to b200SampleAncestralStates.  The histories are checked against the numpy restatement
(oracle/uniformization.py) fed with the engine's own states, categories, rates and generator: jump counts and event states
equal, event times within 1e-13 and totals within 1e-12 relative, except for a (row, pattern) whose draw lies within
BOUNDARY of a CDF boundary (counted and printed).  The sampled totals are checked against the expectations of
b200SampleMarkovJumps and, on non-reversible generators it refuses, against Van Loan's conditional expectations."""
import ctypes as C
import itertools

import numpy as np
import pytest
from scipy.linalg import expm

from beast_mcmc_b200 import beagle
from oracle import markov_jumps as mj
from oracle import uniformization as un
from test_gpu_ancestral import BOUNDARY, NONE, Case, _shard_resource
from test_gpu_markov_jumps import _create, _registers

pytestmark = pytest.mark.gpu

OUT_OF_RANGE = beagle.BeagleErrorCode.OUT_OF_RANGE_ERROR
NO_IMPLEMENTATION = beagle.BeagleErrorCode.NO_IMPLEMENTATION_ERROR


def _row_lengths(case):
    return np.ascontiguousarray(case.lengths[[r[0] for r in case.rows]])


def _cyclic4():
    """non-reversible 4-state generator with a complex pair: a strong cycle 0 -> 1 -> 2 -> 3 -> 0"""
    off = np.full((4, 4), 0.1) - 0.1 * np.eye(4)
    for i in range(4):
        off[i, (i + 1) % 4] = 1.5
    return off - np.diag(off.sum(axis=1))


def _asymmetric(S, seed):
    rng = np.random.default_rng(seed)
    off = rng.uniform(0.0, 1.0, (S, S)) * (rng.random((S, S)) < 0.6)
    np.fill_diagonal(off, 0.0)
    return off - np.diag(off.sum(axis=1))


def _weights(case, inst, seed=1):
    w = np.random.default_rng(seed).integers(1, 5, case.P).astype(np.float64)
    inst.setPatternWeights(w)
    return w


def _evaluate_with(case, inst, Q):
    """transition matrices expm(Q r_c t) set directly (any generator), then the post-order partials"""
    for node in range(case.N):
        if node != case.root:
            inst.setTransitionMatrix(node, np.concatenate([expm(Q * rc * case.lengths[node]).ravel() for rc in case.rates]))
    flat = []
    for n, a, b in case.ops:
        flat += [n, NONE, NONE, a, a, b, b]
    inst.updatePartials(np.array(flat, dtype=np.int32), len(case.ops), NONE)


def _hist(case, inst, Q, regs, seed=7, drawIndex=0, lengths=None, **kw):
    nb, pr, mi = case.arrays()
    lengths = _row_lengths(case) if lengths is None else lengths
    return inst.sampleSubstitutionHistories(nb, pr, mi, lengths, case.root, 0, 0, 0, Q, regs, seed, drawIndex, **kw)


def _pair_ids(jumps):
    return np.repeat(np.arange(jumps.size), jumps.ravel())


def _assert_matches_oracle(case, got, Q, regs, w, seed, drawIndex, label, lengths=None):
    states, cats, branch, pattern, jumps, times, evStates = got
    lengths = _row_lengths(case) if lengths is None else lengths
    want = un.histories([r[1] for r in case.rows], states, cats, lengths, case.rates, Q, regs, w, seed, drawIndex)
    near = want["margins"] < BOUNDARY
    ok = ~near
    print(f"{label}: N = {want['N']}, {int(jumps.sum())} events, {int(near.sum())} of {near.size} pairs within "
          f"{BOUNDARY:g} of a CDF boundary; smallest margin {want['margins'].min():.3e}")
    assert near.mean() <= 0.01
    assert np.array_equal(jumps[ok], want["jumps"][ok]), label
    assert (jumps[0] == 0).all() and (branch[:, 0] == 0).all()
    assert jumps.sum() == len(times) == len(evStates)
    mine, theirs = ok.ravel()[_pair_ids(jumps)], ok.ravel()[_pair_ids(want["jumps"])]
    assert np.array_equal(evStates[mine], want["eventStates"][theirs]), label
    rel = np.abs(times[mine] - want["times"][theirs]) / np.maximum(np.abs(want["times"][theirs]), 1e-300)
    assert rel.size == 0 or rel.max() <= 1e-13, (label, rel.max())
    okPattern = ok.all(axis=0)
    okRow = ok.all(axis=1)
    pr = np.abs(pattern - want["pattern"])[:, okPattern] / np.maximum(np.abs(want["pattern"][:, okPattern]), 1e-300)
    br = np.abs(branch - want["branch"])[:, okRow] / np.maximum(np.abs(want["branch"][:, okRow]), 1e-300)
    print(f"{label}: worst pattern total {pr.max():.3e}, worst branch total {br.max():.3e} relative")
    assert pr.max() <= 1e-12 and br.max() <= 1e-12, label


@pytest.mark.parametrize("S", [4, 12, 20, 61])
@pytest.mark.parametrize("C", [1, 4])
def test_draws_unchanged_and_histories_match_oracle(S, C):
    T, P = {4: (12, 300), 12: (10, 200), 20: (9, 160), 61: (7, 64)}[S]
    case = Case(S=S, C=C, T=T, P=P, seed=S + C)
    inst = case.create()
    case.evaluate(inst)
    w = _weights(case, inst)
    Q = case.model.infinitesimalMatrix()
    regs = _registers(case, "codon" if S == 61 else "nucleotide")
    got = _hist(case, inst, Q, regs, 2024, 5)
    ref = case.sample(inst, 2024, 5)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    _assert_matches_oracle(case, got, Q, regs, w, 2024, 5, f"S={S} C={C}")
    inst.finalize()


def test_single_precision_matches_oracle():
    case = Case(S=4, C=4, T=16, P=500, seed=41)
    inst = case.create(requirement=beagle.BeagleFlag.PRECISION_SINGLE)
    assert inst.getDetails().getFlags() & beagle.BeagleFlag.PRECISION_SINGLE
    case.evaluate(inst)
    w = _weights(case, inst)
    Q = case.model.infinitesimalMatrix()
    regs = _registers(case, "nucleotide")
    got = _hist(case, inst, Q, regs, 11, 1)
    ref = case.sample(inst, 11, 1)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    _assert_matches_oracle(case, got, Q, regs, w, 11, 1, "single")
    inst.finalize()


def test_sampled_totals_match_markov_jumps_expectations():
    """same seed and draw index: the same end states, and the sampled totals average to the expected ones"""
    case = Case(S=4, C=4, T=12, P=20_000, seed=30)
    inst = case.create()
    case.evaluate(inst)
    Q = case.model.infinitesimalMatrix()
    regs = _registers(case, "nucleotide")
    nb, pr, mi = case.arrays()
    st, ca, _, expected = inst.sampleMarkovJumps(nb, pr, mi, _row_lengths(case), case.root, 0, 0, 0, 0, regs, 9, 3,
                                                 branchCounts=False)
    got = _hist(case, inst, Q, regs, 9, 3, branchCounts=False, events=False)
    assert np.array_equal(got[0], st) and np.array_equal(got[1], ca)
    for g in range(len(regs)):
        d = got[3][g] - expected[g]
        se = d.std(ddof=1) * np.sqrt(case.P)
        print(f"register {g}: sampled {got[3][g].sum():.3f}, expected {expected[g].sum():.3f}, {abs(d.sum()) / se:.2f} SE")
        assert abs(d.sum()) <= 5 * se
    inst.finalize()


def _van_loan_means(case, Q, regs, states, cats, lengths):
    """the exact conditional expectation of every (row, pattern), [G][rows][P]"""
    R, P = len(case.rows), case.P
    out = np.zeros((len(regs), R, P))
    for r in range(1, R):
        a, b = states[case.rows[r][1]], states[r]
        for c, rc in enumerate(case.rates):
            sel = cats == c
            tau = rc * lengths[r]
            Pm = expm(Q * tau)
            for g in range(len(regs)):
                N = mj.van_loan(Q, regs[g], tau) / np.where(Pm > 0, Pm, 1.0)
                out[g, r, sel] = N[a[sel], b[sel]]
    return out


def _complex_instance(case):
    inst = _create(case, requirement=beagle.BeagleFlag.EIGEN_COMPLEX)
    ed = case.model.getEigenDecomposition()
    inst.setEigenDecomposition(0, ed.Evec.ravel(), ed.Ievc.ravel(), np.concatenate([ed.Eval, [0.0, 0.3, -0.3, 0.0]]))
    return inst


def test_non_reversible_generator_is_served():
    Q = _cyclic4()
    assert np.abs(np.linalg.eigvals(Q).imag).max() > 1e-3
    regs = np.stack([Q - np.diag(np.diag(Q)), np.diag([0.0, 1.0, 0.0, 0.0])])
    lib = beagle.load_library()
    # against the restatement
    case = Case(S=4, C=2, T=10, P=300, seed=50, partialTips=0)
    inst = _complex_instance(case)
    _evaluate_with(case, inst, Q)
    w = _weights(case, inst)
    outs = _sentinel_outs(case, len(regs))
    args = (inst.instance, *(np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int)) for a in case.arrays()))
    mjRc = lib.b200SampleMarkovJumps(*args, _row_lengths(case).ctypes.data_as(C.POINTER(C.c_double)), len(case.rows),
                                     case.root, 0, 0, 0, 0, np.ascontiguousarray(regs).ctypes.data_as(C.POINTER(C.c_double)),
                                     len(regs), 1, 0, None, None, None, outs[3].ctypes.data_as(C.POINTER(C.c_double)))
    assert mjRc == NO_IMPLEMENTATION
    got = _hist(case, inst, Q, regs, 4, 2)
    _assert_matches_oracle(case, got, Q, regs, w, 4, 2, "non-reversible")
    inst.finalize()
    # against Van Loan
    case = Case(S=4, C=2, T=8, P=20_000, seed=51, partialTips=0)
    inst = _complex_instance(case)
    _evaluate_with(case, inst, Q)
    states, cats, _, pattern, _, _, _ = _hist(case, inst, Q, regs, 6, 0, branchCounts=False, events=False)
    want = _van_loan_means(case, Q, regs, states, cats, _row_lengths(case)).sum(axis=1)
    for g in range(len(regs)):
        d = pattern[g] - want[g]
        se = d.std(ddof=1) * np.sqrt(case.P)
        print(f"register {g}: sampled {pattern[g].sum():.3f}, Van Loan {want[g].sum():.3f}, {abs(d.sum()) / se:.2f} SE")
        assert abs(d.sum()) <= 5 * se
    inst.finalize()


def test_discrete_trait_shape():
    """S = 12, one category, one pattern, 200 tips, an asymmetric location generator"""
    case = Case(S=12, C=1, T=200, P=1, seed=12)
    Q = _asymmetric(12, 3)
    inst = case.create()
    _evaluate_with(case, inst, Q)
    w = _weights(case, inst)
    regs = np.stack([Q - np.diag(np.diag(Q)), np.diag(np.arange(12) == 2).astype(np.float64)])
    got = _hist(case, inst, Q, regs, 5, 0)
    ref = case.sample(inst, 5, 0)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    _assert_matches_oracle(case, got, Q, regs, w, 5, 0, "discrete trait")
    inst.finalize()


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
    Q = case.model.infinitesimalMatrix()
    regs = _registers(case, "nucleotide")
    rowLengths = np.ascontiguousarray(lengths[[r[0] for r in case.rows]])
    got = _hist(case, inst, Q, regs, 3, 4, lengths=rowLengths)
    fresh = case.create()
    case.evaluate(fresh, lengths)
    ref = _hist(case, fresh, Q, regs, 3, 4, lengths=rowLengths)
    margins = case.oracle_draws(inst, 3, 4)[2]
    ok = ~(margins < BOUNDARY).any(axis=0)
    assert ok.mean() >= 0.99
    assert np.array_equal(got[0][:, ok], ref[0][:, ok]) and np.array_equal(got[4][:, ok], ref[4][:, ok])
    assert np.array_equal(got[3][:, ok], ref[3][:, ok])
    inst.finalize(); fresh.finalize()


def test_repeated_calls_bit_identical_and_zero_lengths_give_no_events():
    case = Case(S=4, C=4, T=20, P=300, seed=32)
    inst = case.create()
    case.evaluate(inst)
    _weights(case, inst)
    Q = case.model.infinitesimalMatrix()
    regs = _registers(case, "nucleotide")
    a, b = _hist(case, inst, Q, regs, 1, 0), _hist(case, inst, Q, regs, 1, 0)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert a[4].sum() > 0
    c = _hist(case, inst, Q, regs, 1, 1)
    assert not np.array_equal(a[4], c[4])
    lengths = _row_lengths(case).copy()
    zero = np.arange(len(lengths)) % 3 == 1
    lengths[zero] = 0.0
    z = _hist(case, inst, Q, regs, 1, 0, lengths=lengths)
    assert np.array_equal(z[0], a[0]) and (z[4][zero] == 0).all() and (z[2][:, zero] == 0).all()
    inst.finalize()


def _sentinel_outs(case, G, events=64):
    R = len(case.rows)
    return [np.full((R, case.P), -7, np.int32), np.full(case.P, -7, np.int32), np.full((G, R), -7.0),
            np.full((G, case.P), -7.0), np.full((R, case.P), -7, np.int32), np.full(1, -7, np.int64),
            np.full(events, -7.0), np.full(events, -7, np.int32)]


def _raw_call(lib, inst, case, Q, regs, lengths, outs, capacity=None, nb=None, pr=None, mi=None, root=None, w=0, f=0, r=0,
              G=None, Qptr=True, regsPtr=True, lengthsPtr=True, seed=1, drawIndex=0):
    a_nb, a_pr, a_mi = case.arrays()
    ip = lambda a: np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int))
    dp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))
    ipo = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_int))
    lp = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_longlong))
    nb = a_nb if nb is None else nb
    if capacity is None:
        capacity = 0 if outs[6] is None else len(outs[6])
    return lib.b200SampleSubstitutionHistories(
        inst.instance, ip(nb), ip(a_pr if pr is None else pr), ip(a_mi if mi is None else mi),
        dp(lengths) if lengthsPtr else None, len(nb), case.root if root is None else root, w, f, r,
        dp(Q) if Qptr else None, dp(regs) if regsPtr else None, len(regs) if G is None else G, seed, drawIndex,
        ipo(outs[0]), ipo(outs[1]), dp(outs[2]), dp(outs[3]), ipo(outs[4]), capacity, lp(outs[5]), dp(outs[6]),
        ipo(outs[7]))


def _small_case():
    case = Case(S=4, C=2, T=8, P=40, seed=33)
    return case, np.ascontiguousarray(case.model.infinitesimalMatrix()), np.ascontiguousarray(_registers(case, "nucleotide"))


def test_null_output_combinations_write_only_what_was_asked():
    case, Q, regs = _small_case()
    inst = case.create()
    case.evaluate(inst)
    lengths = _row_lengths(case)
    lib = beagle.load_library()
    probe = _sentinel_outs(case, len(regs))
    assert _raw_call(lib, inst, case, Q, regs, lengths, probe[:6] + [None, None]) == 0
    total = int(probe[5][0])
    assert 0 < total < 2000
    full = _sentinel_outs(case, len(regs), total)
    assert _raw_call(lib, inst, case, Q, regs, lengths, full) == 0
    assert full[5][0] == total and full[4].sum() == total
    for mask in itertools.product([False, True], repeat=8):
        outs = _sentinel_outs(case, len(regs), total)
        ask = [o if m else None for o, m in zip(outs, mask)]
        rc = _raw_call(lib, inst, case, Q, regs, lengths, ask, capacity=total)
        if (mask[6] or mask[7]) and not mask[5]:
            assert rc == OUT_OF_RANGE, mask
            assert all((o == -7).all() for o in outs), mask
            continue
        assert rc == 0, mask
        for o, m, ref in zip(outs, mask, full):
            assert np.array_equal(o, ref) if m else (o == -7).all(), mask
    inst.finalize()


def test_event_capacity_protocol():
    case, Q, regs = _small_case()
    inst = case.create()
    case.evaluate(inst)
    lengths = _row_lengths(case)
    lib = beagle.load_library()
    sizing = _sentinel_outs(case, len(regs))
    sizing[6] = sizing[7] = None
    assert _raw_call(lib, inst, case, Q, regs, lengths, sizing) == 0
    total = int(sizing[5][0])
    exact = _sentinel_outs(case, len(regs), total)
    assert _raw_call(lib, inst, case, Q, regs, lengths, exact) == 0
    assert exact[5][0] == total and np.array_equal(exact[4], sizing[4])
    small = _sentinel_outs(case, len(regs), total)
    assert _raw_call(lib, inst, case, Q, regs, lengths, small, capacity=total - 1) == OUT_OF_RANGE
    assert small[5][0] == total
    assert (small[6] == -7).all() and (small[7] == -7).all()
    assert all(np.array_equal(x, y) for x, y in zip(small[:5], exact[:5]))
    inst.finalize()


@pytest.mark.parametrize("S,P,g", [(4, 301, 3), (4, 2, 3), (20, 97, 2)])
def test_sharded_instance_matches_single_device(S, P, g):
    case = Case(S=S, C=2, T=10, P=P, seed=16 + P)
    res = _shard_resource(list(range(g)))
    whole, sharded = case.create(), case.create(resource=res)
    assert sharded.getDetails().getResourceNumber() == res
    Q = case.model.infinitesimalMatrix()
    regs = _registers(case, "nucleotide")
    w = np.random.default_rng(2).integers(1, 5, P).astype(np.float64)
    for inst in (whole, sharded):
        case.evaluate(inst)
        inst.setPatternWeights(w)
    a, b = _hist(case, whole, Q, regs, 21, 2), _hist(case, sharded, Q, regs, 21, 2)
    for k in (0, 1, 3, 4, 5, 6):
        assert np.array_equal(a[k], b[k]), k
    assert np.allclose(a[2], b[2], rtol=1e-12, atol=0)
    lib = beagle.load_library()
    outs = _sentinel_outs(case, len(regs), len(a[5]))
    assert _raw_call(lib, sharded, case, np.ascontiguousarray(Q), np.ascontiguousarray(regs), _row_lengths(case), outs,
                     capacity=len(a[5]) - 1, seed=21, drawIndex=2) == OUT_OF_RANGE
    assert outs[5][0] == len(a[5]) and (outs[6] == -7).all() and np.array_equal(outs[4], a[4])
    whole.finalize(); sharded.finalize()


def test_errors_return_their_code_and_launch_nothing():
    case = Case(S=4, C=4, T=20, P=300, seed=17, partialTips=0)
    inst = case.create()
    lib = beagle.load_library()
    Q = np.ascontiguousarray(case.model.infinitesimalMatrix())
    regs = np.ascontiguousarray(_registers(case, "nucleotide"))
    lengths = _row_lengths(case)
    G, R = len(regs), len(case.rows)
    case.evaluate(inst)
    out = np.zeros(1)
    inst.calculateRootLogLikelihoods(np.array([case.root], np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32),
                                     np.array([NONE], np.int32), 1, out)
    probe = _sentinel_outs(case, G)
    assert _raw_call(lib, inst, case, Q, regs, lengths, probe[:6] + [None, None]) == 0
    before = _sentinel_outs(case, G, int(probe[5][0]))
    assert _raw_call(lib, inst, case, Q, regs, lengths, before) == 0
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

    def rate(i, j, v):
        x = Q.copy()
        x[i, j] = v
        return dict(Q=x)

    rowSum = Q.copy()
    rowSum[1, 2] += 1e-6
    offNegative = Q.copy()
    offNegative[0, 1], offNegative[0, 2] = -0.01, offNegative[0, 2] + offNegative[0, 1] + 0.01
    bad = [(OUT_OF_RANGE, dict(pr=selfParent)), (OUT_OF_RANGE, dict(root=-1)), (OUT_OF_RANGE, dict(w=10_000)),
           (OUT_OF_RANGE, dict(f=-1)), (OUT_OF_RANGE, dict(r=10_000)), (OUT_OF_RANGE, dict(r=-1)),
           (OUT_OF_RANGE, dict(lengthsPtr=False)), (OUT_OF_RANGE, lens(3, -0.1)), (OUT_OF_RANGE, lens(R - 1, np.nan)),
           (OUT_OF_RANGE, lens(1, np.inf)), (OUT_OF_RANGE, dict(regsPtr=False)), (OUT_OF_RANGE, dict(G=0)),
           (OUT_OF_RANGE, dict(G=9)), (OUT_OF_RANGE, dict(Qptr=False)), (OUT_OF_RANGE, rate(2, 3, np.nan)),
           (OUT_OF_RANGE, rate(1, 1, np.inf)), (OUT_OF_RANGE, dict(Q=rowSum)), (OUT_OF_RANGE, dict(Q=offNegative)),
           (OUT_OF_RANGE, dict(capacity=-1)), (OUT_OF_RANGE, dict(noCount=True)),
           (NO_IMPLEMENTATION, lens(2, 800.0 / float(np.max(-np.diag(Q)) * np.max(case.rates))))]
    for code, kw in bad:
        outs = _sentinel_outs(case, G, len(before[6]))
        ask = list(outs)
        if kw.pop("noCount", False):
            ask[5] = None
        L = kw.pop("lengths", lengths)
        q = kw.pop("Q", Q)
        assert _raw_call(lib, inst, case, q, regs, L, ask, **kw) == code, kw
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
    # back at the original lengths, a valid call gives what it gave before the refusals; row 0's length is not read
    inst.updateTransitionMatrices(0, np.array([node], np.int32), None, None, case.lengths[[node]], 1)
    case.evaluate(inst)
    after = _sentinel_outs(case, G, len(before[6]))
    assert _raw_call(lib, inst, case, Q, regs, lens(0, np.nan)["lengths"], after) == 0
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    inst.finalize()


def test_zero_generator_and_large_state_count():
    case = Case(S=4, C=2, T=8, P=50, seed=18)
    inst = case.create()
    case.evaluate(inst)
    regs = np.stack([np.diag([1.0, 0.0, 0.0, 0.0])])
    states, _, _, pattern, jumps, times, _ = _hist(case, inst, np.zeros((4, 4)), regs, 2, 0)
    assert jumps.sum() == 0 and len(times) == 0
    # Q = 0: no events, each branch spends its whole tau in the parent's state
    tau = _row_lengths(case)[1:, None] * case.rates[_hist(case, inst, np.zeros((4, 4)), regs, 2, 0)[1]][None, :]
    want = (tau * (states[[r[1] for r in case.rows[1:]]] == 0)).sum(axis=0)
    assert np.allclose(pattern[0], want, rtol=1e-12, atol=1e-15)
    inst.finalize()
    big = Case(S=200, C=1, T=3, P=4, seed=19, partialTips=0)
    inst = big.create()
    big.evaluate(inst)
    Q = np.ascontiguousarray(big.model.infinitesimalMatrix())
    regs = np.ascontiguousarray(np.eye(200)[None])
    outs = _sentinel_outs(big, 1)
    assert _raw_call(beagle.load_library(), inst, big, Q, regs, _row_lengths(big), outs) == NO_IMPLEMENTATION
    assert all((o == -7).all() for o in outs)
    inst.finalize()
