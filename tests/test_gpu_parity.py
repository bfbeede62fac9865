"""GPU parity tests: the CUDA engine, called through the C ABI exactly as BEAST's delegate calls
BEAGLE, against (a) the reference's golden values, (b) the numpy oracle on seeded inputs.

Tolerance: north_star's bar is <= 1e-10 relative on the root log-likelihood (fp64 both sides;
differences come from FMA contraction, exp/log implementations and reduction order only).
"""
import math

import numpy as np
import pytest

import helpers as H
from beast_mcmc_b200 import beagle
from harness import evomodel as em, treedatalikelihood as tdl
from test_gpu_virtual_cherries import NONE, Case, _with_env

pytestmark = pytest.mark.gpu

REL = 1e-10
GPU = beagle.BeagleFactory.loadBeagleInstance
S_ = tdl.PartialsRescalingScheme


def _fmt(x):
    return f"{x:.5f}"


def _delegate(tree, pats, model, site, factory, **kw):
    res = [1, 0] if factory is GPU else None
    return tdl.BeagleDataLikelihoodDelegate(tree, pats, model, site, factory, resourceList=res, **kw)


def _pair(tree, pats, model, site, **kw):
    g = _delegate(tree, pats, model, site, GPU, **kw)
    o = _delegate(tree, pats, model, site, H.oracle_factory(report_flags=0), **kw)   # same traversal order
    return g, o


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


# ---- (a) the reference's own golden vectors ----------------------------------------------------
@pytest.mark.parametrize("name", list(H.primate_cases().keys()))
def test_primates_golden(name):
    model, site, expected = H.primate_cases()[name]
    d = _delegate(H.primate_tree(), H.primate_patterns(), model, site, GPU, delayRescalingUntilUnderflow=False)
    assert d.getOptimalTraversalType() == "REVERSE_LEVEL_ORDER"      # instance does not report FRAMEWORK_CPU
    like = tdl.TreeDataLikelihood(d, H.primate_tree())
    assert _fmt(like.getLogLikelihood()) == _fmt(expected)
    d.finalize()


@pytest.mark.parametrize("name", list(H.primate_cases_legacy().keys()))
def test_primates_golden_legacy_likelihood_test(name):
    """The ten values of LikelihoodTest.java:106-341 (other parameters, the older site-model rate rule), alternately with
    and without rescaling."""
    model, site, expected = H.primate_cases_legacy()[name]
    scheme = S_.ALWAYS if len(name) % 2 else S_.NONE
    d = _delegate(H.primate_tree(), H.primate_patterns(), model, site, GPU, rescalingScheme=scheme,
                  delayRescalingUntilUnderflow=False)
    assert _fmt(tdl.TreeDataLikelihood(d, H.primate_tree()).getLogLikelihood()) == _fmt(expected)
    d.finalize()


@pytest.mark.parametrize("k", [0, 1, 2])
def test_msat_hand_calculated_values_to_1e10(k):
    """MsatFullLikelihoodTest.java:181-189 through the C ABI: 3 states on the 4-state kernel (S < 4), 4 states, one pattern;
    the reference asserts 1e-10."""
    tree, pats, model, site, expected = H.msat_cases()[k]
    for scheme in (S_.NONE, S_.ALWAYS):
        d = _delegate(tree, pats, model, site, GPU, rescalingScheme=scheme, delayRescalingUntilUnderflow=False)
        assert abs(tdl.TreeDataLikelihood(d, tree).getLogLikelihood() - expected) <= 1e-10
        d.finalize()


def test_tiny_test_golden():
    tree, pats, model, site, expected = H.tiny_case()
    d = _delegate(tree, pats, model, site, GPU, rescalingScheme=S_.NONE)
    assert _fmt(tdl.TreeDataLikelihood(d, tree).getLogLikelihood()) == _fmt(expected)
    d.finalize()


def test_primates_ambiguity_partials():
    model, site, expected = H.primate_cases()["GTRGI"]
    d = _delegate(H.primate_tree(), H.primate_patterns(), model, site, GPU, useAmbiguities=True,
                  stateSetFn=em.nucleotide_state_set)
    assert _fmt(tdl.TreeDataLikelihood(d, H.primate_tree()).getLogLikelihood()) == _fmt(expected)
    d.finalize()


# ---- (b) oracle parity on seeded synthetic inputs ----------------------------------------------
@pytest.mark.parametrize("tips,patterns,cats,states", [
    (8, 33, 1, 4), (50, 257, 4, 4), (50, 1000, 2, 4), (33, 500, 5, 4), (20, 300, 8, 4), (12, 100, 13, 4),
    (16, 200, 1, 20), (16, 130, 4, 20), (10, 96, 1, 61), (9, 70, 2, 61), (12, 64, 3, 7), (6, 40, 1, 2),
    (10, 64, 40, 4),       # more than 32 categories: 4-state data on the generic block walk
    (6, 40, 1, 70),        # state count without a tensor-path template instance (FMA block walk)
    (7, 48, 2, 30),        # NT = 4 tensor path
])
@pytest.mark.parametrize("scheme", [S_.NONE, S_.ALWAYS])
def test_oracle_parity(tips, patterns, cats, states, scheme):
    tree, pats, model, site = H.synthetic_case(tips, patterns, cats, seed=tips + patterns, stateCount=states)
    g, o = _pair(tree, pats, model, site, rescalingScheme=scheme, delayRescalingUntilUnderflow=False)
    lg = tdl.TreeDataLikelihood(g, tree).getLogLikelihood()
    lo = tdl.TreeDataLikelihood(o, tree).getLogLikelihood()
    assert math.isfinite(lo)
    assert _rel(lg, lo) <= REL, (lg, lo)
    # per-pattern values and every internal node's partials agree too
    assert np.allclose(g.getSiteLogLikelihoods(), o.getSiteLogLikelihoods(), rtol=1e-10, atol=1e-12)
    for node in range(tree.tipCount, tree.nodeCount):
        pg, po = g.getPartials(node), o.getPartials(node)
        # relative agreement, with an absolute floor for entries that are pure cancellation residue
        # of P(t) at tiny rate*time (|P_ij| ~ 1e-13): exp() ulp differences dominate there
        assert np.allclose(pg, po, rtol=1e-9, atol=1e-13 * po.max()), node
    g.finalize()


@pytest.mark.parametrize("log_scalers", [False, True])
def test_scalers_raw_and_log(log_scalers):
    tree, pats, model, site = H.synthetic_case(40, 300, 4, seed=3)
    flag = beagle.BeagleFlag.SCALERS_LOG if log_scalers else 0
    g = _delegate(tree, pats, model, site, GPU, rescalingScheme=S_.ALWAYS, delayRescalingUntilUnderflow=False,
                  preferenceFlags=flag)
    o = _delegate(tree, pats, model, site, H.oracle_factory(extra_flags=flag, report_flags=0),
                  rescalingScheme=S_.ALWAYS, delayRescalingUntilUnderflow=False)
    lg = tdl.TreeDataLikelihood(g, tree).getLogLikelihood()
    lo = tdl.TreeDataLikelihood(o, tree).getLogLikelihood()
    assert _rel(lg, lo) <= REL
    a, b = np.zeros(pats.patternCount), np.zeros(pats.patternCount)
    idx = g.scaleBufferIndices[3]
    g.beagle.getLogScaleFactors(idx, a)
    o.beagle.getLogScaleFactors(o.scaleBufferIndices[3], b)
    assert np.allclose(a, b, rtol=1e-12, atol=1e-13)
    g.finalize()


def test_underflow_protocol_deep_tree():
    """Deep tree: unscaled evaluation underflows -> -Inf -> BEAST switches scaling on and retries
    (BDLD:946-996).  The re-enactment must converge to the oracle's scaled value."""
    tree, pats, model, site = H.synthetic_case(700, 48, 4, seed=9, rootHeight=3000.0)
    g, o = _pair(tree, pats, model, site, rescalingScheme=S_.DYNAMIC, delayRescalingUntilUnderflow=True)
    tg, to = tdl.TreeDataLikelihood(g, tree), tdl.TreeDataLikelihood(o, tree)
    lg, lo = tg.getLogLikelihood(), to.getLogLikelihood()
    assert g.everUnderflowed and o.everUnderflowed and g.useScaleFactors
    assert math.isfinite(lg) and _rel(lg, lo) <= REL, (lg, lo)
    g.finalize()


def test_mcmc_reenactment_store_restore():
    """A short MCMC-like walk: change a node height, evaluate incrementally, accept or reject
    (restore), and compare every step with the oracle driven by the identical call sequence
    and with a from-scratch full evaluation (MarkovChain.java:336-372 self-check)."""
    tree, pats, model, site = H.synthetic_case(60, 500, 4, seed=21)
    tg, to = tree.copy(), tree.copy()
    g, o = _pair(tg, pats, model, site, rescalingScheme=S_.DYNAMIC, delayRescalingUntilUnderflow=True)
    like_g, like_o = tdl.TreeDataLikelihood(g, tg), tdl.TreeDataLikelihood(o, to)
    assert _rel(like_g.getLogLikelihood(), like_o.getLogLikelihood()) <= REL
    rng = np.random.default_rng(0)
    for step in range(25):
        node = int(rng.integers(tree.tipCount, tree.nodeCount - 1))      # internal, not the root
        lo_h = max(tg.height[c] for c in tg.child[node])
        hi_h = tg.height[tg.parent[node]]
        new_h = lo_h + (hi_h - lo_h) * rng.uniform(0.05, 0.95)
        accept = rng.random() < 0.5
        for like, t in ((like_g, tg), (like_o, to)):
            like.storeState()
            old = t.height[node]
            t.height[node] = new_h
            like.updateNodeAndChildren(node)
            val = like.getLogLikelihood()
            if not accept:
                t.height[node] = old
                like.restoreState()
            like._last = val
        assert _rel(like_g._last, like_o._last) <= REL, step
        assert _rel(like_g.getLogLikelihood(), like_o.getLogLikelihood()) <= REL
    # full re-evaluation from scratch equals the incrementally maintained value
    fresh = _delegate(tg, pats, model, site, GPU, rescalingScheme=S_.NONE)
    assert _rel(tdl.TreeDataLikelihood(fresh, tg).getLogLikelihood(), like_g.getLogLikelihood()) <= REL
    g.finalize()
    fresh.finalize()


def test_walk_variants_agree():
    """Matrix-form FMA walk: planned order == caller order, bitwise (same arithmetic).  The eigen-form walk (the default:
    P x evaluated as V (e * (V^-1 x)), walk4e.cu) in its orders and tilings agrees with it to rounding."""
    import os
    tree, pats, model, site = H.synthetic_case(120, 700, 4, seed=4)
    keys = ("B200_REORDER", "B200_EIGEN_WALK", "B200_WALK_R")

    def run(**env):
        for k, v in env.items():
            os.environ[k] = v
        try:
            d = _delegate(tree, pats, model, site, GPU, rescalingScheme=S_.ALWAYS, delayRescalingUntilUnderflow=False)
            v = tdl.TreeDataLikelihood(d, tree).getLogLikelihood()
            d.finalize()
            return v
        finally:
            for k in keys:
                os.environ.pop(k, None)

    vals = [run(B200_EIGEN_WALK="0", B200_REORDER=r) for r in ("0", "1")]
    assert all(v == vals[0] for v in vals), vals
    # eigen form: asynchronous operand staging (k_walk4p) in both op orders and several tilings
    eigen = [run(), run(B200_REORDER="0"), run(B200_WALK_R="2"), run(B200_WALK_R="1")]
    assert all(_rel(v, vals[0]) <= 1e-13 for v in eigen), (eigen, vals[0])
    # same arithmetic whatever the order or the tiling: bit-identical
    assert len(set(eigen)) == 1, eigen


@pytest.mark.parametrize("R", [1, 2, 4])
def test_window_walk_bit_equal_to_staged_walk(R, capfd):
    """At CP <= 8 an aligned list runs on the staged walk k_walk4p, a list with pattern windows (by partition) on
    k_walk4e<CP, R, false>, whose compact tips pick their P column from a per-warp shared-memory table.  Both take the
    same products in the same order: one partition over every pattern gives the internal partials of the plain list bit for
    bit.  CP = 4; B200_WALK_R and B200_THIN_R1=0 fix the tiling R of every phase."""
    case = Case(T=64, P=1000, C=4, seed=17)
    env = {"B200_WALK_R": str(R), "B200_THIN_R1": "0", "B200_BEAGLE_DEBUG": "1"}

    def run(by_partition):
        inst = case.create(True)
        if by_partition:
            inst.setPatternPartitions(1, np.zeros(case.P, dtype=np.int32))
        case.matrices(inst, [n for n in range(case.N) if n != case.root])
        if by_partition:
            flat = []
            for n, a, b in case.ops:
                flat += [n, NONE, NONE, a, case.mat(a), b, case.mat(b), 0, NONE]
            inst.updatePartialsByPartition(np.array(flat, dtype=np.int32), len(case.ops))
        else:
            case.update(inst, case.ops)
        out = [case.partials(inst, n) for n, _, _ in case.ops]
        inst.finalize()
        return out

    staged = _with_env(env, lambda: run(False))
    assert "staged walk" in capfd.readouterr().err
    window = _with_env(env, lambda: run(True))
    assert "staged walk" not in capfd.readouterr().err
    for (n, _, _), a, b in zip(case.ops, staged, window):
        assert np.array_equal(a, b), n


def test_by_partition_equals_separate_instances():
    """updatePartialsByPartition / calculateRootLogLikelihoodsByPartition on one instance equals
    the sum over single-partition instances (MPDLD:744-1207 route; self-consistency pin)."""
    tree, pats, model, site = H.synthetic_case(30, 400, 4, seed=13)
    cut = 150
    model2 = em.HKY(3.0, np.array([0.2, 0.3, 0.3, 0.2]))
    site2 = em.GammaSiteRateModel(shape=1.3, gammaCategoryCount=4)
    parts = [em.Patterns(pats.states[:, :cut], pats.weights[:cut]), em.Patterns(pats.states[:, cut:], pats.weights[cut:])]
    models, sites = [model, model2], [site, site2]
    separate = []
    for k in range(2):
        d = _delegate(tree, parts[k], models[k], sites[k], GPU, rescalingScheme=S_.NONE)
        separate.append(tdl.TreeDataLikelihood(d, tree).getLogLikelihood())
        d.finalize()

    N, nodeCount = tree.tipCount, tree.nodeCount
    b = GPU(N, nodeCount, N, 4, pats.patternCount, 2, 2 * nodeCount, 4, 2 * N, [1, 0], 0, 0)
    for t in range(N):
        b.setTipStates(t, pats.states[t])
    b.setPatternWeights(pats.weights)
    b.setPatternPartitions(2, np.array([0] * cut + [1] * (pats.patternCount - cut), dtype=np.int32))
    like = tdl.TreeDataLikelihood.__new__(tdl.TreeDataLikelihood)     # reuse the traversal only
    like.tree, like.traversalType, like.updateNode = tree, "POST_ORDER", np.ones(nodeCount, dtype=bool)
    like._dispatch()
    for k in range(2):
        e = models[k].getEigenDecomposition()
        b.setEigenDecomposition(k, e.Evec, e.Ievc, e.Eval)
        b.setCategoryRatesWithIndex(k, sites[k].getCategoryRates())
        b.setCategoryWeights(k, sites[k].getCategoryProportions())
        b.setStateFrequencies(k, models[k].getFrequencies())
    nb = len(like.branchOperations)
    eig, rate, prob, lens = [], [], [], []
    for k in range(2):
        for node, t in like.branchOperations:
            eig.append(k); rate.append(k); prob.append(node + k * nodeCount); lens.append(t)
    b.updateTransitionMatricesWithMultipleModels(np.array(eig, dtype=np.int32), np.array(rate, dtype=np.int32),
                                                 np.array(prob, dtype=np.int32), None, None, np.array(lens), 2 * nb)
    ops = []
    for node, c1, c2 in like.nodeOperations:
        for k in range(2):
            ops += [node, -1, -1, c1, c1 + k * nodeCount, c2, c2 + k * nodeCount, k, -1]
    b.updatePartialsByPartition(np.array(ops, dtype=np.int32), len(ops) // 9)
    byPart, total = np.zeros(2), np.zeros(1)
    root = np.array([tree.root, tree.root], dtype=np.int32)
    b.calculateRootLogLikelihoodsByPartition(root, np.array([0, 1], dtype=np.int32), np.array([0, 1], dtype=np.int32),
                                             np.array([-1, -1], dtype=np.int32), np.array([0, 1], dtype=np.int32), 2, 1,
                                             byPart, total)
    assert _rel(byPart[0], separate[0]) <= REL and _rel(byPart[1], separate[1]) <= REL
    assert _rel(total[0], sum(separate)) <= REL

    # same list with per-partition rescaling (MPDLD:972-1017): scaleWrite per node, cumulative buffer per partition
    internal = [node for node, _, _ in like.nodeOperations]
    ops = []
    for node, c1, c2 in like.nodeOperations:
        for k in range(2):
            ops += [node, node - N, -1, c1, c1 + k * nodeCount, c2, c2 + k * nodeCount, k, -1]
    b.updatePartialsByPartition(np.array(ops, dtype=np.int32), len(ops) // 9)
    cum = [2 * N - 2, 2 * N - 1]
    for k in range(2):
        b.resetScaleFactorsByPartition(cum[k], k)
        b.accumulateScaleFactorsByPartition(np.array([n - N for n in internal], dtype=np.int32), len(internal), cum[k], k)
    b.calculateRootLogLikelihoodsByPartition(root, np.array([0, 1], dtype=np.int32), np.array([0, 1], dtype=np.int32),
                                             np.array(cum, dtype=np.int32), np.array([0, 1], dtype=np.int32), 2, 1,
                                             byPart, total)
    assert _rel(byPart[0], separate[0]) <= REL and _rel(byPart[1], separate[1]) <= REL
    b.finalize()


def test_pattern_sharding_sums_to_whole():
    """Patterns.java:142-169 block sharding over instances: sum of shard log-Ls == unsharded."""
    tree, pats, model, site = H.synthetic_case(40, 1003, 4, seed=17)
    whole = _delegate(tree, pats, model, site, GPU, rescalingScheme=S_.NONE)
    lw = tdl.TreeDataLikelihood(whole, tree).getLogLikelihood()
    for shards in (2, 4, 8):
        tot = 0.0
        for k in range(shards):
            d = _delegate(tree, pats.subSet(k, shards), model, site, GPU, rescalingScheme=S_.NONE)
            tot += tdl.TreeDataLikelihood(d, tree).getLogLikelihood()
            d.finalize()
        assert _rel(tot, lw) <= REL
    whole.finalize()


def test_transition_matrices_match_oracle_incl_complex():
    rng = np.random.default_rng(5)
    S, C = 5, 3
    # a non-reversible generator with complex eigenvalues, real block form as Colt/BEAST produce it
    q = rng.uniform(0.05, 1.0, (S, S)); q[0, 1] = 3.0; q[1, 2] = 3.0; q[2, 0] = 3.0
    np.fill_diagonal(q, 0.0); np.fill_diagonal(q, -q.sum(axis=1))
    lam, v = np.linalg.eig(q)
    order, used = [], set()
    evec = np.zeros((S, S)); evr = np.zeros(S); evi = np.zeros(S)
    col = 0
    for k in range(S):
        if k in used:
            continue
        if abs(lam[k].imag) < 1e-12:
            evec[:, col] = v[:, k].real; evr[col] = lam[k].real; col += 1
        else:
            j = [m for m in range(S) if m != k and m not in used and abs(lam[m] - np.conj(lam[k])) < 1e-9][0]
            used.add(j)
            evec[:, col] = v[:, k].real; evec[:, col + 1] = v[:, k].imag
            evr[col] = evr[col + 1] = lam[k].real
            evi[col] = lam[k].imag; evi[col + 1] = -lam[k].imag
            col += 2
        used.add(k)
    ievc = np.linalg.inv(evec)
    evals = np.concatenate([evr, evi])
    from scipy.linalg import expm
    rates = np.array([0.3, 1.0, 1.7])
    lens = np.array([0.01, 0.2, 1.5, 0.0])
    b = GPU(3, 5, 3, S, 16, 1, 8, C, 0, [1, 0], 0, beagle.BeagleFlag.EIGEN_COMPLEX)
    o = H.oracle_factory()(3, 5, 3, S, 16, 1, 8, C, 0, None, 0, beagle.BeagleFlag.EIGEN_COMPLEX)
    for inst in (b, o):
        inst.setEigenDecomposition(0, evec, ievc, evals)
        inst.setCategoryRates(rates)
        inst.updateTransitionMatrices(0, np.arange(4, dtype=np.int32), None, None, lens, 4)
    for k in range(4):
        mg, mo = np.zeros(C * S * S), np.zeros(C * S * S)
        b.getTransitionMatrix(k, mg)
        o.getTransitionMatrix(k, mo)
        assert np.allclose(mg, mo, rtol=1e-12, atol=1e-15)
        for c in range(C):
            assert np.allclose(mg.reshape(C, S, S)[c], expm(q * lens[k] * rates[c]), atol=1e-12)
    b.finalize()


def test_matrix_convolution_and_addition():
    """convolve/addTransitionMatrices (epoch models, SubstitutionModelDelegate.java:303-470): P(t1) x P(t2) == P(t1+t2)."""
    tree, pats, model, site = H.synthetic_case(6, 40, 3, seed=2, stateCount=7)
    S, C = 7, 3
    b = GPU(6, 11, 6, S, pats.patternCount, 1, 8, C, 0, [1, 0], 0, 0)
    o = H.oracle_factory()(6, 11, 6, S, pats.patternCount, 1, 8, C, 0, None, 0, 0)
    e = model.getEigenDecomposition()
    got = []
    for inst in (b, o):
        inst.setEigenDecomposition(0, e.Evec, e.Ievc, e.Eval)
        inst.setCategoryRates(site.getCategoryRates())
        inst.updateTransitionMatrices(0, np.array([0, 1, 2], dtype=np.int32), None, None, np.array([0.03, 0.07, 0.10]), 3)
        inst.convolveTransitionMatrices(np.array([0], dtype=np.int32), np.array([1], dtype=np.int32), np.array([3], dtype=np.int32), 1)
        inst.addTransitionMatrices(np.array([0], dtype=np.int32), np.array([1], dtype=np.int32), np.array([4], dtype=np.int32), 1)
        m = [np.zeros(C * S * S) for _ in range(3)]
        for k, idx in enumerate((2, 3, 4)):
            inst.getTransitionMatrix(idx, m[k])
        got.append(m)
    assert np.allclose(got[0][1], got[0][0], rtol=1e-12, atol=1e-14)          # Chapman-Kolmogorov
    for x, y in zip(got[0], got[1]):
        assert np.allclose(x, y, rtol=1e-12, atol=1e-15)
    b.finalize()


def test_set_get_roundtrips_and_errors():
    b = GPU(4, 7, 4, 4, 37, 2, 14, 3, 8, [1, 0], 0, 0)
    rng = np.random.default_rng(2)
    x = rng.random(3 * 37 * 4)
    b.setPartials(5, x)
    y = np.zeros_like(x)
    b.getPartials(5, beagle.NONE, y)
    assert np.array_equal(x, y)
    m = rng.random(3 * 16)
    b.setTransitionMatrix(9, m)
    m2 = np.zeros_like(m)
    b.getTransitionMatrix(9, m2)
    assert np.array_equal(m, m2)
    st = rng.integers(0, 6, 37).astype(np.int32)
    b.setTipStates(2, st)
    st2 = np.zeros(37, dtype=np.int32)
    b.getTipStates(2, st2)
    assert np.array_equal(np.minimum(st, 4), st2)
    with pytest.raises(beagle.BeagleException) as e:
        b.updatePartials(np.array([99, -1, -1, 0, 0, 1, 1], dtype=np.int32), 1, -1)
    assert e.value.errCode == beagle.BeagleErrorCode.OUT_OF_RANGE_ERROR
    # empty op list is legal (BDLD:904 may pass operationCount == 0)
    b.updatePartials(np.zeros(7, dtype=np.int32), 0, -1)
    b.finalize()


def test_nan_signalling():
    """A NaN sum returns FLOATING_POINT (-8) from the C ABI; the jar/our mirror lets it through and
    BEAST checks isNaN itself (BDLD:946)."""
    lib = beagle.load_library()
    b = GPU(2, 3, 2, 4, 8, 1, 4, 1, 2, [1, 0], 0, 0)
    b.setPartials(2, np.full(8 * 4, np.nan))
    b.setCategoryWeights(0, np.ones(1))
    b.setStateFrequencies(0, np.full(4, 0.25))
    out = np.zeros(1)
    import ctypes as C
    one = (C.c_int * 1)
    rc = lib.beagleCalculateRootLogLikelihoods(b.instance, one(2), one(0), one(0), one(-1), 1,
                                               out.ctypes.data_as(C.POINTER(C.c_double)))
    assert rc == beagle.BeagleErrorCode.FLOATING_POINT_ERROR and math.isnan(out[0])
    b.finalize()


# ---- full-size, size-independent properties (BASELINE.json configs[1]) -------------------------
def test_full_size_properties():
    """1000 taxa x 10,000 patterns, GTR+G4 (synthetic tip data, random states): (i) sharded sum ==
    whole, (ii) scaled == unscaled, (iii) pattern-weight linearity, (iv) oracle on a 256-pattern slice."""
    N, P = 1000, 10000
    tree = em.Tree.coalescent(N, 0.1, 20240924)
    rng = np.random.default_rng(1)
    base = rng.integers(0, 4, P)
    states = ((base[None, :] + (rng.random((N, P)) < 0.08) * rng.integers(1, 4, (N, P))) % 4).astype(np.int32)
    pats = em.Patterns(states, rng.integers(1, 9, P).astype(np.float64))
    model = em.GTR(1.0, 4.0, 0.7, 1.2, 5.0, 1.0, np.array([0.30, 0.22, 0.24, 0.24]))
    site = em.GammaSiteRateModel(shape=0.5, gammaCategoryCount=4)
    d = _delegate(tree, pats, model, site, GPU, rescalingScheme=S_.NONE)
    like = tdl.TreeDataLikelihood(d, tree)
    whole = like.getLogLikelihood()
    sites = d.getSiteLogLikelihoods()
    assert math.isfinite(whole)
    assert _rel(float(np.dot(sites, pats.weights)), whole) <= 1e-12
    d2 = _delegate(tree, pats, model, site, GPU, rescalingScheme=S_.ALWAYS, delayRescalingUntilUnderflow=False)
    assert _rel(tdl.TreeDataLikelihood(d2, tree).getLogLikelihood(), whole) <= REL
    d2.finalize()
    tot = 0.0
    for k in range(4):
        dk = _delegate(tree, pats.subSet(k, 4), model, site, GPU, rescalingScheme=S_.NONE)
        tot += tdl.TreeDataLikelihood(dk, tree).getLogLikelihood()
        dk.finalize()
    assert _rel(tot, whole) <= REL
    sl = em.Patterns(np.ascontiguousarray(states[:, 4000:4256]), pats.weights[4000:4256].copy())
    o = _delegate(tree, sl, model, site, H.oracle_factory(report_flags=0), rescalingScheme=S_.NONE)
    lo = tdl.TreeDataLikelihood(o, tree).getLogLikelihood()
    assert _rel(float(np.dot(sites[4000:4256], sl.weights)), lo) <= REL
    d.finalize()


@pytest.mark.parametrize("name", ["benchmark1_xml", "benchmark2_xml"])
def test_reference_benchmark_alignments(name):
    """The reference's own benchmark inputs (examples/Benchmarks/benchmark{1,2}.xml, committed as pattern fixtures):
    engine == C restatement of the reference algorithm, unscaled and rescaled, on the full alignment."""
    import sys
    sys.path.insert(0, H.ROOT)
    import bench
    from oracle import cpu
    from beast_mcmc_b200 import build
    build.build_oracle()
    w, tree, pats, model, site = bench.build_workload(name, 0, {})
    vals = []
    for factory, res in ((GPU, [1, 0]), (cpu.factory(threads=4), None)):
        for scheme in (S_.NONE, S_.ALWAYS):
            d = tdl.BeagleDataLikelihoodDelegate(tree, pats, model, site, factory, resourceList=res, rescalingScheme=scheme,
                                                 delayRescalingUntilUnderflow=False)
            vals.append(tdl.TreeDataLikelihood(d, tree).getLogLikelihood())
            d.finalize()
    assert math.isfinite(vals[3])
    assert _rel(vals[1], vals[3]) <= REL, vals          # engine rescaled == oracle rescaled
    if math.isfinite(vals[2]):                          # benchmark1 (1441 taxa) underflows unscaled, as it does in BEAST
        assert _rel(vals[3], vals[2]) <= REL and _rel(vals[0], vals[2]) <= REL, vals
    else:
        assert not math.isfinite(vals[0])


def test_concurrent_instances_from_threads():
    """CompoundLikelihood drives one instance per pool thread concurrently (CompoundLikelihood.java:63-82,198-241):
    instances must not share mutable state.  Four instances evaluated from four Python threads (ctypes drops the
    GIL inside the library) give exactly their serial values."""
    import threading
    cases = [H.synthetic_case(30 + 7 * k, 400 + 50 * k, 4, seed=40 + k) for k in range(4)]
    serial = []
    for tree, pats, model, site in cases:
        d = _delegate(tree, pats, model, site, GPU, rescalingScheme=S_.ALWAYS, delayRescalingUntilUnderflow=False)
        serial.append(tdl.TreeDataLikelihood(d, tree).getLogLikelihood())
        d.finalize()
    results = [[] for _ in cases]

    def work(k):
        tree, pats, model, site = cases[k]
        d = _delegate(tree, pats, model, site, GPU, rescalingScheme=S_.ALWAYS, delayRescalingUntilUnderflow=False)
        like = tdl.TreeDataLikelihood(d, tree)
        for _ in range(15):
            like.makeDirty()
            results[k].append(like.getLogLikelihood())
        d.finalize()

    threads = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    for k in range(4):
        assert len(results[k]) == 15 and all(v == serial[k] for v in results[k]), (k, serial[k], results[k][:3])


def test_plan_cache_hits_and_invalidation():
    """Identical op lists are served from the plan cache; a buffer changing kind (setTipStates / setPartials on a tip)
    or different lists must not be.  Every value equals the cache-less engine."""
    import os
    tree, pats, model, site = H.synthetic_case(90, 300, 4, seed=77)      # > 64 operations: planned lists, not the fused route

    def run(cache, graphs="1"):
        os.environ["B200_PLAN_CACHE"] = cache
        os.environ["B200_GRAPHS"] = graphs
        try:
            d = _delegate(tree.copy(), pats, model, site, GPU, rescalingScheme=S_.NONE)
        finally:
            os.environ.pop("B200_PLAN_CACHE", None)
            os.environ.pop("B200_GRAPHS", None)
        like = tdl.TreeDataLikelihood(d, d and tree)
        out = []
        for _ in range(10):                                 # same list, alternating parities -> cache hits, then graph replays
            like.makeDirty()
            out.append(like.getLogLikelihood())
        like.updateNodeAndChildren(tree.tipCount + 3)       # a different (short) list
        out.append(like.getLogLikelihood())
        # tip 0 becomes a partials buffer (all-ones = missing data), then the full list again: the cached plan of
        # that list would read stale compact states
        d.beagle.setPartials(0, np.ones(pats.patternCount * 4 * site.getCategoryCount()))
        like.makeDirty()
        out.append(like.getLogLikelihood())
        d.beagle.setTipStates(0, pats.states[0])
        like.makeDirty()
        out.append(like.getLogLikelihood())
        d.finalize()
        return out

    a, b, c = run("4"), run("0"), run("4", graphs="0")
    assert a == b == c, (a, b, c)
    assert len(set(a[:10])) == 1 and a[12] == a[0] and a[11] != a[0]


def test_graph_replay_follows_substitution_model_moves():
    """A cached plan replayed as a CUDA graph carries V / V^-1 of the list's eigen system BY VALUE in its kernel nodes.  When
    the substitution model moves (new eigen decomposition, same operation list) the captured launches must be patched
    (cudaGraphExecKernelNodeSetParams) or re-captured -- never replayed stale.  Checked against the oracle driven by the same
    calls, and bit-equal to the same engine without graphs."""
    import os

    def run(graphs):
        tree, pats, model, site = H.synthetic_case(90, 300, 4, seed=78)      # > 64 operations: planned lists
        os.environ["B200_GRAPHS"] = graphs
        try:
            g, o = _pair(tree, pats, model, site, rescalingScheme=S_.NONE)
        finally:
            os.environ.pop("B200_GRAPHS", None)
        like_g, like_o = tdl.TreeDataLikelihood(g, tree), tdl.TreeDataLikelihood(o, tree)
        out = []
        for step in range(24):
            if step >= 6 and step % 3 != 2:                 # two moves, one repeat, ...
                model.rates = model.rates.copy()
                model.rates[1] = 2.0 + 0.37 * step          # the A<->G rate: a new eigen system, same lists
                model.rates[4] = 3.0 + 0.11 * step
                model._eigen = None
            for like in (like_g, like_o):
                like.makeDirty()
            vg, vo = like_g.getLogLikelihood(), like_o.getLogLikelihood()
            assert _rel(vg, vo) <= REL, (step, vg, vo)
            out.append(vg)
        g.finalize()
        return out

    a, b = run("1"), run("0")
    assert a == b
    assert len(set(a)) > 10
