"""Pre-order partials + edge derivatives (SURVEY.md 8f rank 1), oracle level (CPU):
the defining identity  sum_c w_c sum_j pre[node]*post[node] = site likelihood  at every node, and the
analytic branch-length gradient against central finite differences of the log-likelihood -- the same
analytic-vs-numeric check the reference's tests/TestXML/testHkyGradient.xml family performs."""
import numpy as np
import pytest

import helpers as H
from harness import treedatalikelihood as tdl


def gradient_and_fd(factory, tree, pats, model, site, resourceList=None, eps=1e-6, nodes=None):
    d = tdl.BeagleDataLikelihoodDelegate(tree, pats, model, site, factory, resourceList=resourceList,
                                         rescalingScheme=tdl.PartialsRescalingScheme.NONE, usePreOrder=True)
    like = tdl.TreeDataLikelihood(d, tree)
    base = like.getLogLikelihood()
    g = tdl.DiscreteTraitBranchRateDelegate(tree, d, model)
    grad = g.getGradient()
    order = [n for n in range(tree.nodeCount) if n != tree.root]
    fd = {}
    tree.branchRate = np.ones(tree.nodeCount)
    for n in (nodes if nodes is not None else order):
        L = tree.branchLength(n)
        vals = []
        for sgn in (+1, -1):
            tree.branchRate[n] = (L + sgn * eps) / L
            like.updateNodeAndChildren(n); like.updateNode[:] = True; like.likelihoodKnown = False
            vals.append(like.getLogLikelihood())
        tree.branchRate[n] = 1.0
        fd[n] = (vals[0] - vals[1]) / (2 * eps)
    like.updateNode[:] = True; like.likelihoodKnown = False
    like.getLogLikelihood()
    return d, g, base, dict(zip(order, grad)), fd


@pytest.mark.parametrize("states,cats", [(4, 1), (4, 4), (20, 2)])
def test_oracle_preorder_identity_and_gradient(states, cats):
    tree, pats, model, site = H.synthetic_case(12, 60, cats, seed=31 + states, stateCount=states)
    d, g, base, grad, fd = gradient_and_fd(H.oracle_factory(), tree, pats, model, site)
    b = d.beagle
    site_l = np.exp(d.getSiteLogLikelihoods())
    w = site.getCategoryProportions()
    for node in range(tree.nodeCount):
        pre = b.partials[g.getPreOrderPartialIndex(node)]
        post = b._post_as_partials(d.getPartialBufferIndex(node))
        lik = sum(w[c] * (pre[c] * post[c]).sum(axis=1) for c in range(len(w)))
        assert np.allclose(lik, site_l, rtol=1e-11), node
    for n, v in fd.items():
        assert abs(grad[n] - v) <= 2e-5 * max(1.0, abs(v)), (n, grad[n], v)


# ---- the CUDA engine through the C ABI ---------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("states,cats,tips,patterns", [(4, 1, 10, 70), (4, 4, 40, 300), (4, 5, 16, 100), (20, 2, 12, 90),
                                                       (61, 1, 8, 64), (7, 3, 9, 50), (4, 2, 10, 97), (4, 8, 12, 301),
                                                       (4, 13, 9, 61), (4, 24, 8, 45), (4, 40, 8, 33), (9, 2, 8, 70),
                                                       (30, 2, 8, 70)])
def test_gpu_preorder_matches_oracle_and_finite_differences(states, cats, tips, patterns):
    from beast_mcmc_b200 import beagle
    tree, pats, model, site = H.synthetic_case(tips, patterns, cats, seed=5 + states + tips, stateCount=states)
    some = [n for n in range(tree.nodeCount) if n != tree.root][::3]
    dg, gg, base_g, grad_g, fd_g = gradient_and_fd(beagle.BeagleFactory.loadBeagleInstance, tree, pats, model, site,
                                                    resourceList=[1, 0], nodes=some)
    do, go, base_o, grad_o, _ = gradient_and_fd(H.oracle_factory(report_flags=0), tree, pats, model, site, nodes=[])
    assert abs(base_g - base_o) <= 1e-10 * abs(base_o)
    for n in grad_o:
        assert abs(grad_g[n] - grad_o[n]) <= 1e-9 * max(1.0, abs(grad_o[n])), (n, grad_g[n], grad_o[n])
    for n, v in fd_g.items():
        assert abs(grad_g[n] - v) <= 5e-5 * max(1.0, abs(v)), (n, grad_g[n], v)
    # pre-order partials themselves, every node
    size = pats.patternCount * states * cats
    for node in range(tree.nodeCount):
        a, b = np.zeros(size), np.zeros(size)
        dg.beagle.getPartials(gg.getPreOrderPartialIndex(node), -1, a)
        do.beagle.getPartials(go.getPreOrderPartialIndex(node), -1, b)
        assert np.allclose(a, b, rtol=1e-9, atol=1e-13 * b.max()), node
    # per-pattern derivatives and the squared sums
    nodes = [n for n in range(tree.nodeCount) if n != tree.root]
    post = np.asarray([dg.getPartialBufferIndex(n) for n in nodes], dtype=np.int32)
    pre = np.asarray([gg.getPreOrderPartialIndex(n) for n in nodes], dtype=np.int32)
    der = np.full(len(nodes), gg.firstDerivativeMatrixIndex, dtype=np.int32)
    outs = []
    for d_, b_ in ((dg, dg.beagle), (do, do.beagle)):
        per, s1, s2 = np.zeros(len(nodes) * pats.patternCount), np.zeros(len(nodes)), np.zeros(len(nodes))
        b_.calculateEdgeDifferentials(post, pre, der, np.zeros(1, dtype=np.int32), len(nodes), per, s1, s2)
        outs.append((per, s1, s2))
    for x, y in zip(outs[0], outs[1]):
        assert np.allclose(x, y, rtol=1e-8, atol=1e-10)
    # transpose round trip
    m, mt, mtt = np.zeros(cats * states * states), np.zeros(cats * states * states), np.zeros(cats * states * states)
    dg.beagle.getTransitionMatrix(0, m)
    dg.beagle.transposeTransitionMatrices(np.array([0], dtype=np.int32), np.array([1], dtype=np.int32), 1)
    dg.beagle.getTransitionMatrix(1, mt)
    assert np.array_equal(mt.reshape(cats, states, states), np.transpose(m.reshape(cats, states, states), (0, 2, 1)))
    dg.finalize()


# ---- cross-product differentials (substitution-parameter gradients) -------------------------------------
def cross_products_and_fd(factory, tree, pats, model, site, resourceList=None, eps=1e-6):
    """Returns the S x S cross products and the finite-difference value of d logL / d log(alpha), alpha a common
    factor on every branch length: with pre and post at the child end of a branch, dP/d alpha = t Q P exactly, so
    sum_ij cross[i][j] Q[i][j] must equal it (AbstractLogAdditiveSubstitutionModelGradient.java:220-227)."""
    d = tdl.BeagleDataLikelihoodDelegate(tree, pats, model, site, factory, resourceList=resourceList,
                                         rescalingScheme=tdl.PartialsRescalingScheme.NONE, usePreOrder=True)
    like = tdl.TreeDataLikelihood(d, tree)
    like.getLogLikelihood()
    g = tdl.SubstitutionModelCrossProductDelegate(tree, d, model)
    cross = g.getCrossProducts()
    vals = []
    for sgn in (+1, -1):
        tree.branchRate = np.full(tree.nodeCount, 1.0 + sgn * eps)
        like.updateNode[:] = True; like.likelihoodKnown = False
        vals.append(like.getLogLikelihood())
    tree.branchRate = np.ones(tree.nodeCount)
    like.updateNode[:] = True; like.likelihoodKnown = False
    like.getLogLikelihood()
    return d, g, cross, (vals[0] - vals[1]) / (2 * eps)


@pytest.mark.parametrize("states,cats", [(4, 1), (4, 4), (20, 2)])
def test_oracle_cross_products_contract_to_scale_derivative(states, cats):
    tree, pats, model, site = H.synthetic_case(11, 50, cats, seed=77 + states, stateCount=states)
    d, g, cross, fd = cross_products_and_fd(H.oracle_factory(), tree, pats, model, site)
    total = float((cross * model.infinitesimalMatrix()).sum())
    assert abs(total - fd) <= 2e-6 * max(1.0, abs(fd)), (total, fd)
    # the call adds to what the caller passes in
    again = np.ones(states * states)
    zero = np.zeros(1, dtype=np.int32)
    nodes = [n for n in range(tree.nodeCount) if n != tree.root]
    d.beagle.calculateCrossProductDifferentials(
        np.asarray([d.getPartialBufferIndex(n) for n in nodes], dtype=np.int32),
        np.asarray([g.getPreOrderPartialIndex(n) for n in nodes], dtype=np.int32), zero, zero,
        np.asarray([tree.branchLength(n) for n in nodes]), len(nodes), again, None)
    assert np.allclose(again - 1.0, cross.reshape(-1), rtol=1e-12, atol=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("states,cats,tips,patterns", [(4, 1, 10, 70), (4, 4, 40, 700), (4, 5, 16, 100), (20, 2, 12, 90),
                                                       (61, 2, 8, 75), (7, 3, 9, 50), (70, 1, 5, 40), (4, 13, 10, 300),
                                                       (16, 2, 8, 70), (30, 2, 8, 70), (3, 4, 9, 80), (40, 2, 6, 40)])
def test_gpu_cross_products_match_oracle(states, cats, tips, patterns):
    from beast_mcmc_b200 import beagle
    tree, pats, model, site = H.synthetic_case(tips, patterns, cats, seed=3 + states + tips, stateCount=states)
    dg, gg, cross_g, fd = cross_products_and_fd(beagle.BeagleFactory.loadBeagleInstance, tree, pats, model, site,
                                                resourceList=[1, 0])
    do, go, cross_o, _ = cross_products_and_fd(H.oracle_factory(report_flags=0), tree, pats, model, site)
    scale = np.abs(cross_o).max()
    assert np.allclose(cross_g, cross_o, rtol=1e-9, atol=1e-12 * scale)
    total = float((cross_g * model.infinitesimalMatrix()).sum())
    assert abs(total - fd) <= 5e-6 * max(1.0, abs(fd))
    # accumulate semantics + subset of branches with tip (compact-state) post buffers only
    tipsOnly = [n for n in range(tree.nodeCount) if tree.isExternal(n)]
    zero = np.zeros(1, dtype=np.int32)
    outs = []
    for d_, g_ in ((dg, gg), (do, go)):
        out = np.full(states * states, 2.0)
        d_.beagle.calculateCrossProductDifferentials(
            np.asarray([d_.getPartialBufferIndex(n) for n in tipsOnly], dtype=np.int32),
            np.asarray([g_.getPreOrderPartialIndex(n) for n in tipsOnly], dtype=np.int32), zero, zero,
            np.asarray([tree.branchLength(n) for n in tipsOnly]), len(tipsOnly), out, None)
        outs.append(out)
    assert np.allclose(outs[0], outs[1], rtol=1e-9, atol=1e-12 * scale)
    dg.finalize()
