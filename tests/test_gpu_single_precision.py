"""PRECISION_SINGLE on 4-state instances: partials stored as fp32, arithmetic in fp64 (DESIGN.md section 4.1).

A single instance behaves as if every partials buffer were written to fp32 memory (round to nearest, subnormal results
flushed to zero) and read back; everything else is the double instance's arithmetic.  A site likelihood is a sum of
non-negative terms, each carrying one factor (1 + delta), |delta| <= u = 2^-24, per stored partials buffer it passes
through (n = internal nodes, plus tips given as partials), so

    |logL_p(single) - logL_p(double)| <= 1.001 n u + 1e-9          (n u <= 1e-3)

for sites whose fp64 partials stay above 2^-126 (without rescaling); 1e-9 covers the fp64 differences between the engine and
the oracle.  Results must not depend on the route a value takes (forwarding, virtual cherries, fusion): every route rounds
at the same points."""
import os

import numpy as np
import pytest

from beast_mcmc_b200 import beagle
from harness import evomodel as em
from harness import treedatalikelihood as tdl
from harness.beagletreelikelihood import BeagleTreeLikelihood, TipPartialsModel
from harness.multipartition import MultiPartitionDataLikelihoodDelegate
import helpers as H

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SINGLE, DOUBLE = beagle.BeagleFlag.PRECISION_SINGLE, beagle.BeagleFlag.PRECISION_DOUBLE
SCALERS_LOG = beagle.BeagleFlag.SCALERS_LOG
NONE = -1
GPU = beagle.BeagleFactory.loadBeagleInstance
S_ = tdl.PartialsRescalingScheme


class _Flags:
    def __init__(self, flags):
        self.flags = flags


def gpu_post_order(*args):
    """the GPU instance, reported to the delegate as a CPU framework: BDLD then sends post-order lists (BDLD:593-599)"""
    inst = GPU(*args)
    flags = inst.getDetails().flags | tdl.FLAG_FRAMEWORK_CPU
    inst.getDetails = lambda: _Flags(flags)
    return inst


def _with_env(env, fn):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return fn()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _create(S, C, pref, req, P=64, resource=1):
    return beagle.BeagleJNIImpl(8, 15, 8, S, P, 1, 14, C, 0, [resource, 0], pref, req)


def _precision(inst):
    f = inst.getDetails().flags
    assert bool(f & SINGLE) != bool(f & DOUBLE), f
    return "single" if f & SINGLE else "double"


# ---- 1. negotiation ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pref,req,small,large", [
    (0, 0, "double", "double"),
    (DOUBLE, 0, "double", "double"),
    (SINGLE | DOUBLE, 0, "double", "double"),
    (SINGLE, 0, "single", "double"),
    (0, SINGLE, "single", None),
    (0, DOUBLE, "double", "double"),
    (SINGLE, DOUBLE, "double", "double"),
])
def test_negotiation(pref, req, small, large):
    inst = _create(4, 4, pref, req)
    assert _precision(inst) == small
    inst.finalize()
    for S, C in ((20, 4), (4, 16)):
        if large is None:
            with pytest.raises(beagle.BeagleException) as e:
                _create(S, C, pref, req)
            assert e.value.errCode == beagle.BeagleErrorCode.NO_RESOURCE_ERROR
        else:
            inst = _create(S, C, pref, req)
            assert _precision(inst) == large
            inst.finalize()


# ---- 2. accuracy against the oracle through the BDLD re-enactment -----------------------------------------------------
def _delegate(tree, pats, model, site, factory, res, scheme, pref=0, **kw):
    return tdl.BeagleDataLikelihoodDelegate(tree, pats, model, site, factory, resourceList=res, rescalingScheme=scheme,
                                            preferenceFlags=pref, **kw)


def _evaluate(d, tree):
    like = tdl.TreeDataLikelihood(d, tree)
    return like.getLogLikelihood(), d.getSiteLogLikelihoods()


def _site_bound(n):
    assert n * U <= 1e-3
    return 1.001 * n * U + 1e-9


@pytest.mark.parametrize("S", [2, 4])
@pytest.mark.parametrize("C", [1, 4, 8])
@pytest.mark.parametrize("scheme", [tdl.PartialsRescalingScheme.NONE, tdl.PartialsRescalingScheme.ALWAYS])
def test_accuracy_against_oracle(S, C, scheme):
    tree, pats, model, site = H.synthetic_case(24, 700, categories=C, seed=31 + C + S, stateCount=S)
    g = _delegate(tree, pats, model, site, beagle.BeagleFactory.loadBeagleInstance, [1, 0], scheme, SINGLE | SCALERS_LOG,
                  delayRescalingUntilUnderflow=False)
    assert g.instanceFlags & SINGLE
    o = _delegate(tree, pats, model, site, H.oracle_factory(), None, scheme, SCALERS_LOG,
                  delayRescalingUntilUnderflow=False)
    (lg, sg), (lo, so) = _evaluate(g, tree), _evaluate(o, tree)
    assert so.min() > -80
    bound = _site_bound(tree.nodeCount - tree.tipCount)
    assert np.max(np.abs(sg - so)) <= bound
    assert abs(lg - lo) <= float(np.sum(pats.weights)) * bound
    # single storage is visible: the values are not the double ones
    assert np.any(sg != so)


def test_accuracy_ambiguity_tip_partials():
    tree, pats, model, site = H.synthetic_case(20, 500, categories=4, seed=41)
    sets = lambda s: np.ones(4) if s >= 4 else np.eye(4)[s]
    g = _delegate(tree, pats, model, site, beagle.BeagleFactory.loadBeagleInstance, [1, 0], tdl.PartialsRescalingScheme.NONE,
                  SINGLE, useAmbiguities=True, stateSetFn=sets)
    o = _delegate(tree, pats, model, site, H.oracle_factory(), None, tdl.PartialsRescalingScheme.NONE, 0,
                  useAmbiguities=True, stateSetFn=sets)
    (_, sg), (_, so) = _evaluate(g, tree), _evaluate(o, tree)
    assert so.min() > -80
    assert np.max(np.abs(sg - so)) <= _site_bound(tree.nodeCount)        # tips are stored partials too


# ---- 3. underflow: fp32 runs out of exponent long before fp64 -----------------------------------------------------------
def test_underflow_switches_on_rescaling():
    # unrelated random tip states on long branches: every site likelihood lies between fp64's and fp32's smallest normals
    tree, _, model, site = H.synthetic_case(80, 8, categories=4, seed=51, rootHeight=1.0)
    rng = np.random.default_rng(52)
    pats = em.Patterns(rng.integers(0, 4, size=(tree.tipCount, 300)).astype(np.int32), np.ones(300), 4)
    make = lambda pref, scheme, **kw: _delegate(tree, pats, model, site, beagle.BeagleFactory.loadBeagleInstance, [1, 0],
                                                scheme, pref, **kw)
    o = _delegate(tree, pats, model, site, H.oracle_factory(), None, tdl.PartialsRescalingScheme.NONE, 0,
                  delayRescalingUntilUnderflow=False)
    _, so = _evaluate(o, tree)
    assert so.min() > -700 and so.max() < -90        # fp64 copes; every site likelihood is below 2^-126
    bound = _site_bound(tree.nodeCount - tree.tipCount)
    # a direct unscaled evaluation: every site is either -inf or right, never finite and wrong
    raw = make(SINGLE, tdl.PartialsRescalingScheme.NONE, delayRescalingUntilUnderflow=False)
    traversal = tdl.TreeDataLikelihood(raw, tree)
    traversal._dispatch()
    with pytest.raises(tdl.LikelihoodUnderflowException):
        raw.calculateLikelihood(traversal.branchOperations, traversal.nodeOperations, tree.root)
    sites = raw.getSiteLogLikelihoods()
    assert np.any(np.isneginf(sites))
    finite = np.isfinite(sites)
    assert np.all(np.isneginf(sites[~finite]))
    assert np.max(np.abs(sites[finite] - so[finite]), initial=0.0) <= bound
    # DYNAMIC scaling, delayed until the first underflow (BEAST's default): only the single delegate needs it
    vals = {}
    for name, pref in (("single", SINGLE), ("double", 0)):
        d = make(pref, tdl.PartialsRescalingScheme.DYNAMIC)
        vals[name] = (tdl.TreeDataLikelihood(d, tree).getLogLikelihood(), d.everUnderflowed)
    assert vals["single"][1] and not vals["double"][1]
    lo = float(np.sum(pats.weights * so))
    assert abs(vals["single"][0] - lo) <= float(np.sum(pats.weights)) * bound
    assert abs(vals["double"][0] - lo) <= float(np.sum(pats.weights)) * 1e-9


# ---- 4. route independence, bit for bit ---------------------------------------------------------------------------------
def _single_run(env, tree, pats, model, site, moves=()):
    def run():
        t = tree.copy()
        d = _delegate(t, pats, model, site, beagle.BeagleFactory.loadBeagleInstance, [1, 0],
                      tdl.PartialsRescalingScheme.NONE, SINGLE)
        like = tdl.TreeDataLikelihood(d, t)
        vals = [like.getLogLikelihood()]
        for node in moves:
            t.height[node] = 0.5 * (max(t.height[c] for c in t.child[node]) + t.height[t.parent[node]])
            like.updateNodeAndChildren(node)
            vals.append(like.getLogLikelihood())
        parts = [d.getPartials(n) for n in range(t.tipCount, t.nodeCount)]
        fused = d.beagle._lib.b200GetFusedLaunches(d.beagle.instance)
        return vals, d.getSiteLogLikelihoods(), parts, fused
    return _with_env(env, run)


@pytest.mark.parametrize("env", [{"B200_VIRTUAL_CHERRIES": "0"}, {"B200_FORWARD": "0"}])
def test_routes_bitwise(env):
    tree, pats, model, site = H.synthetic_case(64, 1000, categories=4, seed=61)
    base = _single_run({}, tree, pats, model, site)
    other = _single_run(env, tree, pats, model, site)
    assert base[0] == other[0]
    assert np.array_equal(base[1], other[1])
    for a, b in zip(base[2], other[2]):
        assert np.array_equal(a, b)
    # every stored value is an fp32 number
    for a in base[2]:
        assert np.array_equal(a, a.astype(np.float32).astype(np.float64))


def test_fused_route_bitwise():
    tree, pats, model, site = H.synthetic_case(64, 1000, categories=4, seed=71)
    moves = (tree.tipCount + 3, tree.tipCount + 9)
    fused = _single_run({}, tree, pats, model, site, moves)
    plain = _single_run({"B200_FUSE": "0"}, tree, pats, model, site, moves)
    assert fused[3] > 0 and plain[3] == 0
    for a, b in zip(fused[2], plain[2]):
        assert np.array_equal(a, b)
    for a, b in zip(fused[0], plain[0]):
        assert abs(a - b) <= 1e-12 * abs(b)


# ---- 5. setPartials / getPartials ------------------------------------------------------------------------------------
def test_set_get_partials_round_to_fp32():
    rng = np.random.default_rng(81)
    inst = _create(4, 4, SINGLE, 0)
    P = 64
    x = rng.uniform(1e-6, 1.0, 4 * P * 4)
    inst.setPartials(9, x)
    out = np.zeros_like(x)
    inst.getPartials(9, NONE, out)
    assert np.array_equal(out, x.astype(np.float32).astype(np.float64))
    inst.finalize()


def test_accuracy_post_order_lists():
    tree, pats, model, site = H.synthetic_case(40, 600, categories=4, seed=37)
    for scheme in (S_.NONE, S_.ALWAYS):
        g = _delegate(tree, pats, model, site, gpu_post_order, [1, 0], scheme, SINGLE, delayRescalingUntilUnderflow=False)
        assert g.getOptimalTraversalType() == "POST_ORDER" and g.instanceFlags & SINGLE
        o = _delegate(tree, pats, model, site, H.oracle_factory(), None, scheme, 0, delayRescalingUntilUnderflow=False)
        (lg, sg), (lo, so) = _evaluate(g, tree), _evaluate(o, tree)
        assert so.min() > -80
        bound = _site_bound(tree.nodeCount - tree.tipCount)
        assert np.max(np.abs(sg - so)) <= bound
        assert abs(lg - lo) <= float(np.sum(pats.weights)) * bound


def test_beagle_tree_likelihood_route():
    """BeagleTreeLikelihood with tip partials (every tip is a stored buffer too) under DYNAMIC scaling"""
    tree, pats, model, site = H.synthetic_case(32, 333, 4, seed=8)
    rng = np.random.default_rng(8)
    noisy = []
    for t in range(tree.tipCount):
        q = np.eye(4)[np.minimum(pats.states[t], 3)] * 0.96 + 0.01
        q[rng.random(pats.patternCount) < 0.05] = 1.0
        noisy.append(q)
    vals = []
    for factory, res, pref in ((GPU, [1, 0], SINGLE), (H.oracle_factory(report_flags=0), None, 0)):
        like = BeagleTreeLikelihood(pats, tree.copy(), model, site, factory, tipStatesModel=TipPartialsModel(noisy),
                                    resourceList=res, rescalingScheme=S_.DYNAMIC, preferenceFlags=pref)
        vals.append(like.getLogLikelihood())
        if factory is GPU:
            assert like.beagle.getDetails().flags & SINGLE
            like.finalize()
    assert abs(vals[0] - vals[1]) <= float(np.sum(pats.weights)) * _site_bound(tree.nodeCount)


# ---- 4b. graph replay across substitution-model moves equals a fresh instance ------------------------------------------
def test_graph_replay_equals_fresh_instance():
    tree, pats, model, site = H.synthetic_case(90, 300, 4, seed=78)          # > 64 operations: planned, cached, replayed
    d = _delegate(tree, pats, model, site, GPU, [1, 0], S_.NONE, SINGLE)
    like = tdl.TreeDataLikelihood(d, tree)
    for step in range(12):
        if step >= 4 and step % 3 != 2:
            model.rates = model.rates.copy()
            model.rates[1] = 2.0 + 0.37 * step
            model.rates[4] = 3.0 + 0.11 * step
            model._eigen = None
        like.makeDirty()
        v = like.getLogLikelihood()
        if step in (5, 7, 11):
            fresh = _delegate(tree, pats, model, site, GPU, [1, 0], S_.NONE, SINGLE)
            vf = tdl.TreeDataLikelihood(fresh, tree).getLogLikelihood()
            assert v == vf, (step, v, vf)
            assert np.array_equal(d.getSiteLogLikelihoods(), fresh.getSiteLogLikelihoods())
            assert np.array_equal(d.getPartials(tree.root), fresh.getPartials(tree.root))
            fresh.beagle.finalize()
    assert d.beagle._lib.b200GetFusedLaunches(d.beagle.instance) == 0
    d.beagle.finalize()


# ---- 5b. getPartials with a scale index: widened, then unscaled in fp64 -------------------------------------------------
def test_get_partials_with_scale_index():
    tree, pats, model, site = H.synthetic_case(40, 500, categories=4, seed=83)
    g = _delegate(tree, pats, model, site, GPU, [1, 0], S_.ALWAYS, SINGLE | SCALERS_LOG, delayRescalingUntilUnderflow=False)
    o = _delegate(tree, pats, model, site, H.oracle_factory(), None, S_.ALWAYS, SCALERS_LOG, delayRescalingUntilUnderflow=False)
    _evaluate(g, tree), _evaluate(o, tree)
    n = tree.nodeCount - tree.tipCount
    out = {}
    for name, d in (("g", g), ("o", o)):
        cum = d.scaleBufferHelper.getOffsetIndex(d.internalNodeCount)
        buf = np.zeros(4 * 4 * pats.patternCount)
        d.beagle.getPartials(d.getPartialBufferIndex(tree.root), cum, buf)
        out[name] = buf
    # each element is a sum of non-negative terms with at most n fp32 roundings
    assert np.all(np.abs(out["g"] - out["o"]) <= (1.001 * n * U + 1e-9) * out["o"])
    assert not np.array_equal(out["g"], out["g"].astype(np.float32).astype(np.float64))   # unscaled after widening


# ---- 6. *ByPartition ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scheme", [S_.NONE, S_.ALWAYS])
def test_by_partition_route(scheme):
    sizes = (37, 333, 90, 51)
    tree, pats, model, site = H.synthetic_case(40, sum(sizes), 4, seed=105)
    cuts = np.cumsum((0,) + sizes)
    parts = [em.Patterns(np.ascontiguousarray(pats.states[:, a:b]), pats.weights[a:b].copy(), 4)
             for a, b in zip(cuts[:-1], cuts[1:])]
    rng = np.random.default_rng(105)
    models = [em.HKY(1.5 + k, rng.dirichlet(np.full(4, 8.0))) for k in range(len(sizes))]
    sites = [em.GammaSiteRateModel(shape=0.4 + 0.3 * k, gammaCategoryCount=4) for k in range(len(sizes))]
    kw = dict(rescalingScheme=scheme, delayRescalingUntilUnderflow=False)
    g = MultiPartitionDataLikelihoodDelegate(tree, parts, models, sites, GPU, resourceList=[1, 0], preferenceFlags=SINGLE, **kw)
    assert g.beagle.getDetails().flags & SINGLE
    o = MultiPartitionDataLikelihoodDelegate(tree, parts, models, sites, H.oracle_factory(report_flags=0), **kw)
    lg, lo = tdl.TreeDataLikelihood(g, tree), tdl.TreeDataLikelihood(o, tree)
    bound = _site_bound(tree.nodeCount - tree.tipCount)
    for evaluation in range(2):
        vg, vo = lg.getLogLikelihood(), lo.getLogLikelihood()
        sg, so = g.getSiteLogLikelihoods(), o.getSiteLogLikelihoods()
        assert so.min() > -80
        assert np.max(np.abs(sg - so)) <= bound
        assert abs(vg - vo) <= float(np.sum(pats.weights)) * bound
        for k, p in enumerate(parts):
            assert abs(g.cachedLogLikelihoodsByPartition[k] - o.cachedLogLikelihoodsByPartition[k]) <= \
                float(np.sum(p.weights)) * bound
        lg.makeDirty()
        lo.makeDirty()
    g.finalize()


# ---- 7. gradients --------------------------------------------------------------------------------------------------------
def _gradient_pair(S, seed, C=4):
    tree, pats, model, site = H.synthetic_case(30, 600, categories=C, seed=seed, stateCount=S)
    out = []
    for factory, res, pref in ((GPU, [1, 0], SINGLE), (H.oracle_factory(), None, 0)):
        d = _delegate(tree, pats, model, site, factory, res, S_.NONE, pref, usePreOrder=True)
        tdl.TreeDataLikelihood(d, tree).getLogLikelihood()
        out.append(d)
    assert out[0].instanceFlags & SINGLE
    return tree, pats, model, out[0], out[1]


@pytest.mark.parametrize("C", [4, 1, 8])
@pytest.mark.parametrize("S", [2, 4])
def test_edge_derivatives_bound(S, C):
    """Per pattern and edge, d_p = num_p / L_p with num_p = sum_c w_c sum_jk pre_cj D_cjk post_ck and
    L_p = sum_c w_c sum_j pre_cj post_cj.  Every pre and post value passed through at most N stored fp32 buffers, so it
    carries a factor (1 + e) with |e| <= 1.001 N u (N = all pre- and post-order buffers; n u << 1 keeps the 1.001).  A term
    of num_p carries two such factors and is bounded by its |.| version, so |dnum| <= 2.002 N u A_p with
    A_p = sum_c w_c sum_jk pre_cj |D_cjk| post_ck; likewise |dL| <= 2.002 N u L_p.  Then
        |dd_p| <= |dnum| / L + |d_p| |dL| / L <= 1.001 u (2N A_p/L_p + 2N |d_p|) <= 1.001 u (3N A_p/L_p + N |d_p|)
    as |d_p| <= A_p / L_p.  1e-9 A_p/L_p covers the fp64 differences from the oracle.  A_p comes from the oracle's
    partials."""
    tree, pats, model, g, o = _gradient_pair(S, 91 + S, C)
    nodes = [n for n in range(tree.nodeCount) if n != tree.root]
    N = (tree.nodeCount - tree.tipCount) + tree.nodeCount
    dg, do = tdl.DiscreteTraitBranchRateDelegate(tree, g, model), tdl.DiscreteTraitBranchRateDelegate(tree, o, model)
    P = pats.patternCount
    per = {}
    for name, d, deleg in (("g", g, dg), ("o", o, do)):
        deleg.simulate()
        deleg.cacheDifferentialMassMatrix()
        post = np.asarray([d.getPartialBufferIndex(n) for n in nodes], dtype=np.int32)
        pre = np.asarray([deleg.getPreOrderPartialIndex(n) for n in nodes], dtype=np.int32)
        der = np.full(len(nodes), deleg.firstDerivativeMatrixIndex, dtype=np.int32)
        per[name] = np.zeros(len(nodes) * P)
        d.beagle.calculateEdgeDifferentials(post, pre, der, np.zeros(1, dtype=np.int32), len(nodes), per[name],
                                            np.zeros(len(nodes)), np.zeros(len(nodes)))
    ob = o.beagle
    w = ob.categoryWeights[0]
    D = ob.matrices[do.firstDerivativeMatrixIndex]
    for e, node in enumerate(nodes):
        post = ob._post_as_partials(o.getPartialBufferIndex(node))
        pre = ob.partials[do.getPreOrderPartialIndex(node)]
        A = sum(w[c] * np.einsum("pj,jk,pk->p", pre[c], np.abs(D[c]), post[c]) for c in range(o.categoryCount))
        L = sum(w[c] * np.einsum("pj,pj->p", pre[c], post[c]) for c in range(o.categoryCount))
        d_o, d_g = per["o"][e * P:(e + 1) * P], per["g"][e * P:(e + 1) * P]
        bound = 1.001 * U * (3 * N * A / L + N * np.abs(d_o)) + 1e-9 * A / L
        assert np.all(np.abs(d_g - d_o) <= bound), (node, np.max(np.abs(d_g - d_o) / bound))


@pytest.mark.parametrize("C", [4, 1, 8])
@pytest.mark.parametrize("S", [2, 4])
def test_cross_products_bound(S, C):
    """out[i][j] = sum_e t_e sum_p w_p (sum_c w_c r_c pre_ci post_cj) / L_p: every term is non-negative, the numerator carries
    two factors (1 + e) and L_p two more, |e| <= 1.001 N u, so each entry is within 1.001 * 4 N u of the oracle's
    (relative), plus 1e-9 for the fp64 differences."""
    tree, pats, model, g, o = _gradient_pair(S, 95 + S, C)
    N = (tree.nodeCount - tree.tipCount) + tree.nodeCount
    xg = tdl.SubstitutionModelCrossProductDelegate(tree, g, model).getCrossProducts()
    xo = tdl.SubstitutionModelCrossProductDelegate(tree, o, model).getCrossProducts()
    assert np.all(np.isfinite(xg)) and np.all(xo >= 0)
    assert np.all(np.abs(xg - xo) <= (1.001 * 4 * N * U + 1e-9) * xo)


def test_pre_order_forwarding_bitwise():
    """pre[parent] forwarded in registers to the first child (B200_FORWARD) is the rounded value the buffer holds"""
    tree, pats, model, site = H.synthetic_case(64, 800, categories=4, seed=99)
    runs = []
    for env in ({}, {"B200_FORWARD": "0"}):
        def run():
            d = _delegate(tree, pats, model, site, GPU, [1, 0], S_.NONE, SINGLE, usePreOrder=True)
            tdl.TreeDataLikelihood(d, tree).getLogLikelihood()
            deleg = tdl.DiscreteTraitBranchRateDelegate(tree, d, model)
            grad = deleg.getGradient()
            pre = []
            for n in range(tree.nodeCount):
                buf = np.zeros(4 * 4 * pats.patternCount)
                d.beagle.getPartials(deleg.getPreOrderPartialIndex(n), NONE, buf)
                pre.append(buf)
            d.beagle.finalize()
            return grad, pre
        runs.append(_with_env(env, run))
    assert np.array_equal(runs[0][0], runs[1][0])
    for a, b in zip(runs[0][1], runs[1][1]):
        assert np.array_equal(a, b)
        assert np.array_equal(a, a.astype(np.float32).astype(np.float64))


# ---- 8. the sharded resource -------------------------------------------------------------------------------------------
def test_sharded_single_equals_mode_a():
    import ctypes
    import torch
    lib = beagle.load_library()
    number = [r.number for r in beagle.BeagleFactory.getResourceDetails() if "pattern-sharded" in r.name]
    assert number
    n = torch.cuda.device_count()
    devices = [k % n for k in range(2)]
    assert lib.b200SetShardDevices((ctypes.c_int * 2)(*devices), 2) == 0
    tree, pats, model, site = H.synthetic_case(100, 1003, 4, seed=21)       # > 64 operations: the planned route on both
    kw = dict(rescalingScheme=S_.NONE, delayRescalingUntilUnderflow=False, preferenceFlags=SINGLE)
    sharded = tdl.BeagleDataLikelihoodDelegate(tree, pats, model, site, GPU, resourceList=[number[0], 0], **kw)
    assert sharded.beagle.getDetails().getResourceNumber() == number[0]
    assert sharded.instanceFlags & SINGLE and not sharded.instanceFlags & DOUBLE
    vs = tdl.TreeDataLikelihood(sharded, tree).getLogLikelihood()
    total = 0.0
    for k in range(2):
        d = tdl.BeagleDataLikelihoodDelegate(tree, pats.subSet(k, 2), model, site, GPU, resourceList=[1, 0], **kw)
        assert d.instanceFlags & SINGLE
        total += tdl.TreeDataLikelihood(d, tree).getLogLikelihood()
        d.finalize()
    assert vs == total, (vs, total)
    sharded.finalize()


def test_cross_products_fewer_than_four_states_double():
    """S < 4 on the 4-state layout takes the generic cross-product kernel (k_cross4 is S = 4 only), in double as in single"""
    tree, pats, model, site = H.synthetic_case(30, 600, categories=4, seed=97, stateCount=2)
    out = []
    for factory, res in ((GPU, [1, 0]), (H.oracle_factory(), None)):
        d = _delegate(tree, pats, model, site, factory, res, S_.NONE, 0, usePreOrder=True)
        tdl.TreeDataLikelihood(d, tree).getLogLikelihood()
        out.append(tdl.SubstitutionModelCrossProductDelegate(tree, d, model).getCrossProducts())
    assert np.allclose(out[0], out[1], rtol=1e-10, atol=0)
