"""The gradient route (updatePrePartials, calculateEdgeDifferentials, calculateCrossProductDifferentials) against the
oracle on every kernel and shape it dispatches to.

Each case drives the engine and oracle/felsenstein.py with the same raw call sequence (``Twin``) and compares node by
node and value by value.  A case's docstring names the route it targets and the dispatch rule that sends it there
(function and condition); the suite does not assert kernel names.

Tolerances are those of the other fp64 gradient tests (tests/test_preorder_oracle.py): partials rtol 1e-9 with an
absolute floor of 1e-13 times the buffer's maximum, per-pattern derivatives rtol 1e-8 / atol 1e-10, cross products
rtol 1e-9 with a floor of 1e-12 times the largest entry.  fp32 cases reuse the derived bounds of
tests/test_gpu_single_precision.py."""
import os

import numpy as np
import pytest

from beast_mcmc_b200 import beagle
from oracle.felsenstein import OracleBeagle
import helpers as H
from test_preorder_oracle import gradient_and_fd

pytestmark = pytest.mark.gpu

NONE = -1
U = 2.0 ** -24
SINGLE = beagle.BeagleFlag.PRECISION_SINGLE
SCALERS_LOG = beagle.BeagleFlag.SCALERS_LOG
I32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)


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


def _close(a, b, rtol=1e-9, floor=1e-13):
    return np.allclose(a, b, rtol=rtol, atol=floor * max(np.abs(b).max(), 1e-300))


class Twin:
    """One engine instance and one oracle instance fed identical calls.

    Buffers: post-order partials of node n at n (tips 0..T-1: compact states with gaps, or tip partials with ambiguity
    sets), pre-order partials of node n at N + n.  Matrix n is P(t) of node n's branch,
    matrices N .. N + nDiff - 1 are distinct differential matrices.  Scale buffers: post-order writes of internal node n
    at n - T, pre-order writes of node n at T - 1 + n, cumulative buffers at 2N and 2N + 1.  Category weights and rates
    sets 0 (the site model's) and 1 (a different set)."""

    def __init__(self, S, C, tips, P, seed, *, pref=0, env=None, partialTips=0.3, rootHeight=0.1, nDiff=3, oracle=True,
                 data=None):
        self.S, self.C, self.P = S, C, P
        self.tree, pats, self.model, self.site = data if data is not None else \
            H.synthetic_case(tips, P, C, seed=seed, stateCount=S, rootHeight=rootHeight)
        tree = self.tree
        self.N, self.T, self.root = N, T, root = tree.nodeCount, tree.tipCount, tree.root
        self.nDiff = nDiff
        rng = np.random.default_rng(seed + 1000)
        states = pats.states.copy()
        states[rng.random(states.shape) < 0.06] = S                                    # gaps
        self.states = states
        self.weights = pats.weights.copy()
        self.partialTips = set(int(t) for t in rng.choice(T, size=int(round(partialTips * T)), replace=False))
        args = (T, 2 * N + 4, T, S, P, 2, N + nDiff, C, 2 * N + 2)
        self.gpu = _with_env(env or {}, lambda: beagle.BeagleJNIImpl(*args, [1, 0], pref, 0))
        self.ora = OracleBeagle(*args, None, pref, 0) if oracle else None
        self.cumPost, self.cumPre = 2 * N, 2 * N + 1
        self.both("setPatternWeights", self.weights)
        for t in range(T):
            if t in self.partialTips:                  # as useAmbiguities does: one-hot rows, ones for a gap, some pairs
                part = np.zeros((P, S))
                known = states[t] < S
                part[np.nonzero(known)[0], states[t][known]] = 1.0
                part[~known] = 1.0
                amb = np.nonzero(known & (rng.random(P) < 0.15))[0]
                part[amb, (states[t][amb] + 1) % S] = 1.0
                self.both("setTipPartials", t, part.reshape(-1))
            else:
                self.both("setTipStates", t, I32(states[t]))
        ed = self.model.getEigenDecomposition()
        self.both("setEigenDecomposition", 0, ed.Evec.reshape(-1), ed.Ievc.reshape(-1), ed.Eval)
        self.both("setStateFrequencies", 0, self.model.getFrequencies())
        self.both("setStateFrequencies", 1, self.model.getFrequencies())
        self.w = [self.site.getCategoryProportions(), rng.dirichlet(np.full(C, 2.0))]
        self.r = [self.site.getCategoryRates(), self.site.getCategoryRates() * rng.uniform(0.5, 1.5, C)]
        for k in range(2):
            self.both("setCategoryWeights", k, self.w[k])
            self.both("setCategoryRatesWithIndex", k, self.r[k])
        self.both("setCategoryRates", self.r[0])
        self.edges = [n for n in range(N) if n != root]
        self.both("updateTransitionMatrices", 0, I32(self.edges), None, None,
                  np.asarray([tree.branchLength(n) for n in self.edges]), len(self.edges))
        Q = self.model.infinitesimalMatrix()
        for k in range(nDiff):                         # a distinct derivative matrix per index: not a multiple of Q
            R = rng.normal(size=(S, S))
            D = np.concatenate([((1.0 + 0.5 * k) * Q + 0.2 * k * R) * rc for rc in self.r[0]])
            self.both("setDifferentialMatrix", N + k, D.reshape(-1))

    def both(self, name, *args):
        getattr(self.gpu, name)(*args)
        if self.ora is not None:
            getattr(self.ora, name)(*args)

    def finalize(self):
        self.gpu.finalize()

    def pre(self, n):
        return self.N + n

    def der(self, n):
        return self.N + n % self.nDiff

    # ---- traversals ------------------------------------------------------------------------------------------------
    def post_order(self, scale=False):
        """internal nodes in numbering order (children first); with ``scale`` every op writes its factor and the list
        accumulates into cumPost.  Returns (engine, oracle) log-likelihoods."""
        ops = []
        for n in range(self.T, self.N):
            c1, c2 = (int(c) for c in self.tree.child[n])
            ops += [n, n - self.T if scale else NONE, NONE, c1, c1, c2, c2]
        cum = self.cumPost if scale else NONE
        if scale:
            self.both("resetScaleFactors", cum)
        self.both("updatePartials", I32(ops), len(ops) // 7, cum)
        out = []
        for b in (self.gpu, self.ora):
            if b is None:
                continue
            v = np.zeros(1)
            b.calculateRootLogLikelihoods(I32([self.root]), I32([0]), I32([0]), I32([cum]), 1, v)
            out.append(float(v[0]))
        return out

    def pre_order_ops(self, scaling=None):
        """(parent, node, sibling) in pre-order (SimulationTreeTraversal), then op tuples; ``scaling(k, node)`` gives
        (destinationScaleWrite, destinationScaleRead) of op k"""
        tree, order, stack = self.tree, [], [(self.root, -1, -1)]
        while stack:
            node, parent, sib = stack.pop()
            if parent >= 0:
                order.append((parent, node, sib))
            if not tree.isExternal(node):
                c1, c2 = int(tree.child[node][0]), int(tree.child[node][1])
                stack.append((c2, node, c1))
                stack.append((c1, node, c2))
        ops = []
        for k, (parent, node, sib) in enumerate(order):
            sw, sr = scaling(k, node) if scaling else (NONE, NONE)
            ops += [self.pre(node), sw, sr, self.pre(parent), node, sib, sib]
        return ops

    def pre_order(self, scaling=None, cum=NONE):
        P, C = self.P, self.C
        self.both("setPartials", self.pre(self.root), np.tile(self.model.getFrequencies(), P * C))
        if cum != NONE:
            self.both("resetScaleFactors", cum)
        ops = self.pre_order_ops(scaling)
        self.both("updatePrePartials", I32(ops), len(ops) // 7, cum)

    # ---- reads -----------------------------------------------------------------------------------------------------
    def partials(self, b, idx, scaleIdx=NONE):
        out = np.zeros(self.P * self.S * self.C)
        b.getPartials(idx, scaleIdx, out)
        return out

    def all_pre(self, b):
        return [self.partials(b, self.pre(n)) for n in range(self.N)]

    def check_pre(self):
        for n in range(self.N):
            a, o = self.partials(self.gpu, self.pre(n)), self.partials(self.ora, self.pre(n))
            assert _close(a, o), (n, np.max(np.abs(a - o) / (np.abs(o) + 1e-300)))

    def edge_derivatives(self, b, nodes, wIdx=1, outs=(True, True, True), der=None):
        count = len(nodes)
        per = np.zeros(count * self.P) if outs[0] else None
        s1 = np.zeros(count) if outs[1] else None
        s2 = np.zeros(count) if outs[2] else None
        b.calculateEdgeDifferentials(I32(nodes), I32([self.pre(n) for n in nodes]),
                                     I32(der if der is not None else [self.der(n) for n in nodes]), I32([wIdx]), count,
                                     per, s1, s2)
        return per, s1, s2

    def check_edges(self, nodes=None, combos=((True, True, True), (True, False, False), (False, True, False),
                                             (False, False, True), (False, False, False))):
        """every null/non-null combination of the three outputs, weights set 1; returns the full engine outputs"""
        nodes = self.edges if nodes is None else nodes
        full = None
        for outs in combos:
            g = self.edge_derivatives(self.gpu, nodes, outs=outs)
            o = self.edge_derivatives(self.ora, nodes, outs=outs)
            for x, y in zip(g, o):
                if y is not None:
                    assert np.allclose(x, y, rtol=1e-8, atol=1e-10), (outs, np.max(np.abs(x - y)))
            if all(outs):
                full = g
        return full

    def cross(self, b, nodes, lengths, rIdx=1, wIdx=0, init=None):
        out = np.zeros(self.S * self.S) if init is None else np.array(init, dtype=np.float64)
        b.calculateCrossProductDifferentials(I32(nodes), I32([self.pre(n) for n in nodes]), I32([rIdx]), I32([wIdx]),
                                             np.asarray(lengths, dtype=np.float64), len(nodes), out, None)
        return out

    def check_cross(self, reps=1):
        """rates set 1 and weights set 1, into a non-zero output; every edge ``reps`` times with distinct lengths
        (count >> the kernels' edge groups).  The oracle runs once per distinct edge at length 1: the result is linear
        in the lengths."""
        E = len(self.edges)
        nodes = np.resize(self.edges, E * reps)
        lengths = np.asarray([self.tree.branchLength(n) for n in nodes]) * (1.0 + 0.37 * (np.arange(E * reps) // E))
        init = np.linspace(-1.0, 2.0, self.S * self.S)
        g = self.cross(self.gpu, nodes, lengths, rIdx=1, wIdx=1, init=init)
        per = {n: self.cross(self.ora, [n], [1.0], rIdx=1, wIdx=1) for n in self.edges}
        o = init + sum(t * per[n] for n, t in zip(nodes, lengths))
        scale = np.abs(o - init).max()
        assert np.allclose(g - init, o - init, rtol=1e-9, atol=1e-12 * scale), np.max(np.abs(g - o)) / scale


# ---- 1. 4-state pre-order on every CP and R ------------------------------------------------------------------------------
CATS = [1, 2, 3, 8, 13, 24, 40]          # matCP 1, 2, 4, 8, 16, 32, and 0 (C > 32: generic walk)
R_ENV = {1: {}, 2: {"B200_WALK_R": "2", "B200_THIN_R1": "0"}, 4: {"B200_WALK_R": "4", "B200_THIN_R1": "0"}}


@pytest.mark.parametrize("P", [301, 1])
@pytest.mark.parametrize("R", [1, 2, 4])
@pytest.mark.parametrize("C", CATS)
def test_preorder4_every_cp_and_r(C, R, P):
    """Route: 4-state pre-order walk k_walk4<CP, R, false, 4, true> (kernels.cu launchWalk4 -> launchWalk4T<CP>), CP =
    matCP = C rounded up to a power of two (beagleCreateInstance); C = 40 has matCP = 0 and takes k_walk_generic
    (launchWalkGeneric, Sp = 4).  R = 1: the default rule of beagleCreateInstance halves walkR while a subtree has fewer
    warps than SMs, and launchWalk4T's thin rule (walks < smCount * 8) picks R = 1 anyway.  R = 2 / 4: B200_WALK_R
    forces walkR and B200_THIN_R1=0 disables the thin rule.  P = 301 leaves a partial last tile for every 32/CP * R,
    P = 1 a tile with one live pattern."""
    tw = Twin(4, C, 12, P, seed=100 + C + R, env=R_ENV[R])
    try:
        lg, lo = tw.post_order()
        assert abs(lg - lo) <= 1e-10 * abs(lo)
        tw.pre_order()
        tw.check_pre()
        tw.check_edges(combos=((True, True, True),))
    finally:
        tw.finalize()


@pytest.mark.parametrize("C,tips,P", [(4, 200, 5000), (24, 64, 2000)])
def test_preorder4_natural_r4(C, tips, P):
    """Route: k_walk4<CP, 4, false, 4, true> by the default rules alone: walkR stays 4 in beagleCreateInstance because
    Ppad / (32/CP * 4) >= smCount (1250 warps at CP = 4, 500 at CP = 32), and the phases of planPreorderPhases are wide
    enough that launchWalk4T's thin rule (walks < smCount * 8) does not apply."""
    tw = Twin(4, C, tips, P, seed=7 + C, partialTips=0.1)
    try:
        lg, lo = tw.post_order()
        assert abs(lg - lo) <= 1e-10 * abs(lo)
        tw.pre_order()
        tw.check_pre()
        tw.check_edges(combos=((True, True, True),))
    finally:
        tw.finalize()


# ---- 2. scaled pre-order lists ------------------------------------------------------------------------------------------
def _pre_scaling(tw, phase):
    """phase 0: ops 1, 4, 7, ... write their own scale buffer.  phase 1 (the list under test): ops 0, 3, 6, ... write
    their own buffer, ops 1, 4, ... read the buffer they wrote in phase 0, the rest neither.  No op reads a buffer
    another op of the same list writes: lists are ordered by their partials dependencies only."""
    written = []

    def scaling(k, node):
        slot = tw.T - 1 + node
        if k % 3 == 1 - phase:
            written.append(slot)
            return slot, NONE
        if phase == 1 and k % 3 == 1:
            return NONE, slot
        return NONE, NONE
    return scaling, written


@pytest.mark.parametrize("log", [False, True])
@pytest.mark.parametrize("S,C", [(4, 4), (20, 2), (70, 1)])
def test_scaled_preorder_list(S, C, log):
    """Route: pre-order ops with destinationScaleWrite / destinationScaleRead (factors a previous list wrote) and a
    cumulative index, on the 4-state walk (k_walk4<4, R, false, 4, true>, matCP = 4), the DMMA walk
    (k_walk_mma<3, .., PRE = true>: Sp = 24, launchWalkGeneric with genericMma) and the FMA generic walk (k_walk_generic:
    Sp = 72 has no DMMA instance).  The walk rescales by the per-pattern maximum and stores the factor (log under
    SCALERS_LOG); accumulateInList adds the written factors' logs to the cumulative buffer after the phases.  Partials,
    every written buffer's and the cumulative buffer's log factors, and the edge derivatives are compared."""
    tw = Twin(S, C, 10, 77, seed=200 + S + C + log, pref=SCALERS_LOG if log else 0)
    try:
        lg, lo = tw.post_order()
        assert abs(lg - lo) <= 1e-10 * abs(lo)
        first, written0 = _pre_scaling(tw, 0)
        tw.pre_order(first)
        scaling, written = _pre_scaling(tw, 1)
        tw.pre_order(scaling, cum=tw.cumPre)
        written += written0
        assert written0 and written
        tw.check_pre()
        for idx in written + [tw.cumPre]:
            a, b = np.zeros(tw.P), np.zeros(tw.P)
            tw.gpu.getLogScaleFactors(idx, a)
            tw.ora.getLogScaleFactors(idx, b)
            assert np.allclose(a, b, rtol=1e-10, atol=1e-12), idx
            if idx != tw.cumPre:
                assert np.any(a != 0.0)
        # a scaled buffer read back with the cumulative index: pre partials times exp(cum)
        n = tw.edges[-1]
        assert _close(tw.partials(tw.gpu, tw.pre(n), tw.cumPre), tw.partials(tw.ora, tw.pre(n), tw.cumPre))
        tw.check_edges(combos=((True, True, True),))
    finally:
        tw.finalize()


@pytest.mark.parametrize("S,C", [(4, 4), (20, 2)])
def test_gradient_on_rescaled_post_order(S, C):
    """Route: edge derivatives on post-order partials rescaled with ALWAYS semantics (every op writes its factor, a
    cumulative buffer for the root).  A per-pattern factor on post[node] (and through the siblings on pre[node])
    multiplies both num_p and L_p, so the derivatives equal the unscaled oracle's."""
    tw = Twin(S, C, 24, 150, seed=300 + S, rootHeight=0.6)
    try:
        lg, lo = tw.post_order(scale=True)
        assert abs(lg - lo) <= 1e-10 * abs(lo)
        tw.pre_order()
        tw.check_pre()
        scaled = tw.check_edges(combos=((True, True, True),))
        lu = tw.post_order(scale=False)
        assert abs(lu[1] - lo) <= 1e-10 * abs(lo)
        tw.pre_order()
        plain = tw.edge_derivatives(tw.ora, tw.edges)
        for x, y in zip(scaled, plain):
            assert np.allclose(x, y, rtol=1e-8, atol=1e-10)
    finally:
        tw.finalize()


# ---- 3. pre-order plan routes, double: oracle and bit-identical to the default route -------------------------------------
@pytest.mark.parametrize("tips,P,env", [
    (512, 96, {}),
    (40, 133, {"B200_PHASE_T": "2", "B200_PHASE_TMIN": "1"}),
    (512, 96, {"B200_PRE_PHASES": "0"}),
    (512, 96, {"B200_FORWARD": "0"}),
    (512, 96, {"B200_LOOKAHEAD_PRE": "0"}),
])
def test_preorder_plan_routes(tips, P, env):
    """Route: beagleUpdatePrePartials -> planAndLaunch.  Default: planPreorderPhases cuts the list into subtree phases,
    pre[parent] read across phases.  B200_PHASE_T=2 forces two-op subtrees on a small tree (many phases).
    B200_PRE_PHASES=0 takes planLevels (one launch per level).  B200_FORWARD=0 stores and reloads pre[parent] instead of
    forwarding it in registers; B200_LOOKAHEAD_PRE=0 drops the look-ahead prefetch.  Each route does the same per-cell
    arithmetic as the default, so its partials and derivatives are bit-identical to it."""
    data = H.synthetic_case(tips, P, 4, seed=400 + tips, stateCount=4)
    runs = []
    for e in (env, {}) if env else (env,):
        tw = Twin(4, 4, tips, P, seed=400 + tips, env=e, oracle=not runs, data=data)
        try:
            tw.post_order()
            tw.pre_order()
            if tw.ora is not None:
                tw.check_pre()
                tw.check_edges(combos=((True, True, True),))
            runs.append((tw.all_pre(tw.gpu), tw.edge_derivatives(tw.gpu, tw.edges)))
        finally:
            tw.finalize()
    if len(runs) == 2:
        for a, b in zip(runs[0][0], runs[1][0]):
            assert np.array_equal(a, b)
        for a, b in zip(runs[0][1], runs[1][1]):
            assert np.array_equal(a, b)


# ---- 4. edge derivatives, every kernel ----------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [255, 256, 257])
@pytest.mark.parametrize("C", CATS)
def test_edge_derivatives4(C, P):
    """Route: k_edge_derivatives4 (launchEdgeDerivatives: partial != nullptr && matCP > 0, edgeDerivativeWorkspace gives
    S = 4 with matCP > 0 a workspace), one block per 256-pattern chunk: P = 255 / 256 / 257 sit on either side of the
    chunk.  C = 40 (matCP = 0, Sp = 4) has no tensor form and takes k_edge_derivatives with the MT[c][k][j] addressing
    of dIndex."""
    tw = Twin(4, C, 8, P, seed=500 + C + P)
    try:
        tw.post_order()
        tw.pre_order()
        tw.check_edges()
    finally:
        tw.finalize()


@pytest.mark.parametrize("S,C,env", [
    (9, 2, {}), (16, 2, {}), (20, 2, {}), (30, 2, {}), (61, 1, {}),
    (3, 4, {}), (40, 2, {}), (70, 1, {}), (70, 6, {}), (20, 2, {"B200_GENERIC_MMA": "0"}),
])
def test_edge_derivatives_generic_layouts(S, C, env):
    """Routes (launchEdgeDerivatives, edgeDerivativeWorkspace): S = 9, 16 -> k_edge_derivatives_mma<2>, 20 -> <3>,
    30 -> <4>, 61 -> <8> (genericMma, matCP = 0, Sp / 8 in 1..4 or 8), P = 100 (P mod 64 != 0) with tip edges.
    k_edge_derivatives (no tensor form): S = 3 (Sp = 4, matCP > 0 but S != 4: dIndex's matCP branch), S = 40 (Sp / 8 = 5)
    and S = 70, C = 1 with D staged in shared memory (C S^2 8 B <= budget); S = 70, C = 6 exceeds the budget and runs
    with stageD = 0, reading D from global memory; B200_GENERIC_MMA=0 sends S = 20 to k_edge_derivatives too."""
    tw = Twin(S, C, 9, 100, seed=600 + S + C, env=env)
    try:
        lg, lo = tw.post_order()
        assert abs(lg - lo) <= 1e-10 * abs(lo)
        tw.pre_order()
        tw.check_edges()
    finally:
        tw.finalize()


# ---- 5. more edges than a grid's y dimension ----------------------------------------------------------------------------
@pytest.mark.parametrize("S,single", [(4, False), (4, True), (20, False)])
def test_edge_count_above_65535(S, single):
    """Route: count > 65535 -> edgeDerivativeWorkspace returns 0 and every state count takes the one-block-per-edge
    k_edge_derivatives (S = 4: dIndex's matCP branch; PRECISION_SINGLE: k_edge_derivatives_f32).  Each copy of an edge is
    computed by one block with the same arithmetic, so copies are bit-identical.  The distinct-edge call takes
    k_edge_derivatives4 / k_edge_derivatives_mma<3>: compared with a tolerance (different summation order)."""
    C = 4 if S == 4 else 2
    tw = Twin(S, C, 10, 37, seed=700 + S + single, pref=SINGLE if single else 0)
    try:
        tw.post_order()
        tw.pre_order()
        E, count = len(tw.edges), 70000
        nodes = np.resize(tw.edges, count)
        per, s1, s2 = tw.edge_derivatives(tw.gpu, nodes)
        per = per.reshape(count, tw.P)
        first = np.arange(count) % E
        assert np.array_equal(per, per[first]) and np.array_equal(s1, s1[first]) and np.array_equal(s2, s2[first])
        dper, ds1, ds2 = tw.edge_derivatives(tw.gpu, tw.edges)
        assert np.allclose(per[:E].reshape(-1), dper, rtol=1e-11, atol=1e-13)
        assert np.allclose(s1[:E], ds1, rtol=1e-11, atol=1e-13 * np.abs(ds1).max())
        assert np.allclose(s2[:E], ds2, rtol=1e-11, atol=1e-13 * np.abs(ds2).max())
        oper, os1, os2 = tw.edge_derivatives(tw.ora, tw.edges)
        if not single:
            assert np.allclose(per[:E].reshape(-1), oper, rtol=1e-8, atol=1e-10)
            assert np.allclose(s1[:E], os1, rtol=1e-8, atol=1e-10)
            assert np.allclose(s2[:E], os2, rtol=1e-8, atol=1e-10)
        else:
            _check_single_edge_bound(tw, per[:E].reshape(-1), oper)
    finally:
        tw.finalize()


def _check_single_edge_bound(tw, got, want):
    """the bound of tests/test_gpu_single_precision.py::test_edge_derivatives_bound: pre and post values each passed
    through at most N stored fp32 buffers (N = internal post-order nodes + all pre-order nodes + the tips given as
    partials), so |dd_p| <= 1.001 u (3 N A_p / L_p + N |d_p|), plus 1e-9 A_p / L_p for the fp64 differences"""
    o, P = tw.ora, tw.P
    N = (tw.N - tw.T) + tw.N + len(tw.partialTips)
    w = o.categoryWeights[1]
    for e, node in enumerate(tw.edges):
        post, pre, D = o._post_as_partials(node), o.partials[tw.pre(node)], o.matrices[tw.der(node)]
        A = sum(w[c] * np.einsum("pj,jk,pk->p", pre[c], np.abs(D[c]), post[c]) for c in range(tw.C))
        L = sum(w[c] * np.einsum("pj,pj->p", pre[c], post[c]) for c in range(tw.C))
        d_o, d_g = want[e * P:(e + 1) * P], got[e * P:(e + 1) * P]
        bound = 1.001 * U * (3 * N * A / L + N * np.abs(d_o)) + 1e-9 * A / L
        assert np.all(np.abs(d_g - d_o) <= bound), (node, np.max(np.abs(d_g - d_o) / bound))


# ---- 6. cross products, every kernel ------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,C,P", [
    (4, 1, 300), (4, 3, 300), (4, 8, 300), (4, 13, 300), (4, 32, 300),
    (8, 2, 100), (16, 2, 100), (20, 2, 100), (30, 2, 100), (61, 1, 100),
    (3, 4, 90), (40, 2, 50), (130, 2, 50),
])
def test_cross_products_every_kernel(S, C, P):
    """Routes (launchCrossProducts, crossGeometry): S = 4 -> k_cross4 (Sp == 4 && S == 4), 256-pattern chunks crossed by
    P = 300; S = 8, 16, 20, 30, 61 -> k_cross_mma<1, 2, 3, 4, 8> (genericMma, Sp % 8 == 0, Sp / 8 in 1..4 or 8);
    S = 3 (Sp = 4 but S != 4), 40 (Sp / 8 = 5) and 130 (S4 / 4 = 33: 1089 4x4 tiles, five passes of the tile loop) ->
    k_cross_generic.  Every edge 30 times with different lengths: count well above the edge groups, so every block runs
    the e += gridDim.y loop.  Rates set 1, weights set 1, added to a non-zero output."""
    tw = Twin(S, C, 8, P, seed=800 + S + C)
    try:
        tw.post_order()
        tw.pre_order()
        tw.check_cross(reps=1)
        tw.check_cross(reps=30)
    finally:
        tw.finalize()


# ---- 7. large discrete-trait state counts -------------------------------------------------------------------------------
@pytest.mark.parametrize("S,C", [(130, 2), (255, 1)])
def test_large_state_count(S, C):
    """Routes at S > 120: the generic walk unstaged (k_walk_generic, stage = 0 in launchWalkGeneric), post- and pre-order;
    k_edge_derivatives with stageD = 0 (C S^2 8 B over the shared-memory budget); k_cross_generic with 5 (S = 130) and
    16 (S = 255) passes of the tile loop.  Log-likelihood, every pre-order partial, the edge derivatives and the cross
    products against the oracle, and the analytic gradient against central finite differences on a few nodes."""
    tw = Twin(S, C, 6, 50, seed=900 + S)
    try:
        lg, lo = tw.post_order()
        assert abs(lg - lo) <= 1e-10 * abs(lo)
        tw.pre_order()
        tw.check_pre()
        tw.check_edges()
        tw.check_cross(reps=3)
    finally:
        tw.finalize()
    tree, pats, model, site = H.synthetic_case(6, 50, C, seed=950 + S, stateCount=S)
    some = [n for n in range(tree.nodeCount) if n != tree.root][::3]
    dg, gg, base_g, grad_g, fd_g = gradient_and_fd(beagle.BeagleFactory.loadBeagleInstance, tree, pats, model, site,
                                                    resourceList=[1, 0], nodes=some)
    _, _, base_o, grad_o, _ = gradient_and_fd(H.oracle_factory(report_flags=0), tree, pats, model, site, nodes=[])
    try:
        assert abs(base_g - base_o) <= 1e-10 * abs(base_o)
        for n in grad_o:
            assert abs(grad_g[n] - grad_o[n]) <= 1e-9 * max(1.0, abs(grad_o[n])), (n, grad_g[n], grad_o[n])
        for n, v in fd_g.items():
            assert abs(grad_g[n] - v) <= 5e-5 * max(1.0, abs(v)), (n, grad_g[n], v)
    finally:
        dg.finalize()
