"""The post-order 4-state walk against the oracle on every route walk4Route (walk4e.cu) dispatches to.

walk4Route picks each phase's kernel family -- matrix form (k_walk4 / k_walk4s), eigen form with per-pattern predicates
(k_walk4e<CP, R, false> / k_walk4es), eigen form without them (k_walk4e<CP, R, true>, CP 16 and 32), staged
(k_walk4p / k_walk4ps) or staged with virtual cherries (k_walk4pv / k_walk4pvs) -- and R, the patterns per thread; the
instance supplies CP (the category count rounded up to a power of two) and the precision.  Every row of CASES names one
such cell and the inputs that send a list there:

  * R: B200_WALK_R forces walkR and B200_THIN_R1=0 switches off the thin-phase rule, so the route no longer depends on the
    SM count or the phase shapes.  The eigen form is built for R = 2 at CP = 4 only (walkR 2 runs R = 4 elsewhere).
  * Matrix: B200_EIGEN_WALK=0, or matrices set with setTransitionMatrix (no eigen system behind them).
  * EigenPredicated: by-partition lists (partition windows start off warp multiples; one partition is one pattern wide),
    and aligned lists at (CP 1, R 4) / (CP 2, R 4) whose Ppad is not a multiple of G * R, G = 32 / CP.
  * EigenAligned: aligned lists at CP 16 and 32.
  * Staged: aligned lists at CP <= 8 with Ppad a multiple of G * R >= 4, B200_VIRTUAL_CHERRIES=0.
  * StagedVirtual: the same with cherries between compact tips; the plan line reports them.
  * Two rows set no knob at all: their routes follow from the default walkR and thin rules.

B200_FUSE=0 keeps short lists off the one-launch incremental evaluation (incr.cu), which is not a walk route.  With
B200_BEAGLE_DEBUG every launched phase logs its kernel and R (api.cu launchPlan); each case asserts that its cell ran.

Every case drives the engine and oracle/felsenstein.py with the same raw calls (Twin of test_gpu_gradient_routes.py) and
checks node by node: a list run three times with new branch lengths (a fresh plan, a cache hit, a graph capture that
replays) and once more after a new eigen system (the captured eigen-form launches are patched in place,
updateWalk4EGraph); buffers outside the list's writes stay bit-identical; by-partition rows update one partition alone and
the other partitions' columns must keep their values; R = 4 rows then run a rescaled list (every other op with an
internal child writes its factor -- never a cherry -- raw and SCALERS_LOG alternating, some with an in-list cumulative
index) and a second list that reads those factors through destinationScaleRead.

Tolerances.  fp64: partials rtol 1e-9 with a floor of 1e-13 times the buffer's maximum, root log-likelihood rel 1e-10,
site log-likelihoods rtol 1e-10 / atol 1e-12, log scale factors rtol 1e-10 / atol 1e-12.  fp32 storage (PRECISION_SINGLE)
keeps fp64 arithmetic and rounds each stored value to fp32: a partials entry of node n is a sum of non-negative terms,
each a product of factors that passed through at most k_n stored buffers (k_n = internal nodes in n's subtree, n
included, plus the tips in it given as partials; a virtual cherry is rounded as if stored), each rounding contributing
(1 + d), |d| <= u = 2^-24.  So

    |x_engine - x_oracle| <= (1.001 k_n u + 1e-9) x_oracle          (k_n u <= 1e-3; 1e-9 covers the fp64 differences)

as long as the values stay above fp32's smallest normal (a few dozen tips on short branches).  Rescaling divides by a
per-pattern maximum computed from the rounded children, so a scaled value also carries the error of its subtree's
factors; the product of the stored value and the factors of its subtree, exp(sum of log factors), does not: it is the
unscaled value and obeys the bound above.  The factors: with D_n the error of the summed log factors of n's subtree,
D_n = error of log max V_n for a node that writes one (|.| <= 1.001 k_n u) and D_c1 + D_c2 otherwise, so every
|D_n| <= 1.001 k_n u, one factor's log is within 2.002 k_n u (+ 1e-9) and the cumulative buffer within 1.001 k_root u
(+ 1e-9)."""
import re
from collections import namedtuple

import numpy as np
import pytest

from beast_mcmc_b200 import beagle
from harness import evomodel as em
from test_gpu_gradient_routes import I32, NONE, SCALERS_LOG, SINGLE, U, Twin, _close

pytestmark = pytest.mark.gpu

MATRIX, EIGEN_PREDICATED, EIGEN_ALIGNED, STAGED, STAGED_VIRTUAL = range(5)     # Walk4Kernel (engine.h)
FAMILY = {MATRIX: "matrix", EIGEN_PREDICATED: "eigen-predicated", EIGEN_ALIGNED: "eigen-aligned", STAGED: "staged",
          STAGED_VIRTUAL: "staged-virtual"}
CATS = {1: 1, 2: 2, 4: 3, 8: 5, 16: 13, 32: 24}       # CP -> a category count below it: idle category lanes
PS = [33, 96, 301, 1000]                              # Ppad 64; Ppad 96 and 320; ~1000

# family, CP, R, single: the cell.  C, S, P, tips: the instance.  lists: "aligned" or "partition" (by-partition lists);
# matrices: "eigen" (updateTransitionMatrices), "set" (setTransitionMatrix); env: the knobs; scale: None, "write" (factors
# accumulated after the list) or "cum" (in-list cumulative index); log: SCALERS_LOG; natural: routes by the default rules
Case = namedtuple("Case", "family cp r single C S P tips lists matrices env scale log natural")


def _ppad(P):
    return -(-P // 32) * 32


def _parts(P):
    """contiguous partitions with boundaries off warp multiples; the first is one pattern wide, the widest an odd count"""
    if P == 1:
        return [1]
    k = (P - 1) // 3 + 2
    k += (P - 1 - k) % 2 == 0
    return [1, k, P - 1 - k]


def _live(P, lists):
    """live patterns of a list's widest pattern window: all of an aligned list, the widest partition of a by-partition
    list (a warp there starts at its partition's first pattern)"""
    return P if lists == "aligned" else max(_parts(P))


def _case(family, cp, r, single, P, *, C=None, S=4, tips=20, lists="aligned", matrices="eigen", scale=None, log=False,
          natural=False, env=None):
    if env is None:
        env = {"B200_WALK_R": str(r), "B200_THIN_R1": "0", "B200_FUSE": "0"}
        if family == MATRIX and matrices == "eigen":
            env["B200_EIGEN_WALK"] = "0"
        if family == STAGED:
            env["B200_VIRTUAL_CHERRIES"] = "0"
    return Case(family, cp, r, single, CATS[cp] if C is None else C, S, P, tips, lists, matrices, env, scale, log, natural)


def _cases():
    rows = []
    k = 0

    def p_for(family, cp, r, lists):
        """the next P of the rotation whose widest window fills every lane and r slot of a warp (G * R patterns) and
        leaves a tail (a warp that is partly live); the staged kernels also need Ppad to be whole warps"""
        nonlocal k
        g_r = 32 // cp * r
        for _ in range(len(PS)):
            P = PS[k % len(PS)]
            k += 1
            live = _live(P, lists)
            if live >= g_r and (live % g_r != 0 or g_r == 1) and (family not in (STAGED, STAGED_VIRTUAL) or _ppad(P) % g_r == 0):
                return P
        raise AssertionError((family, cp, r, lists))

    for single in (False, True):
        cps = [1, 2, 4, 8] if single else [1, 2, 4, 8, 16, 32]
        for cp in cps:
            for r in (1, 2, 4):
                rows.append(_case(MATRIX, cp, r, single, p_for(MATRIX, cp, r, "aligned"),
                                  matrices="set" if r == 2 else "eigen"))
            for r in ((1, 2, 4) if cp == 4 else (1, 4)):
                rows.append(_case(EIGEN_PREDICATED, cp, r, single, p_for(EIGEN_PREDICATED, cp, r, "partition"),
                                  lists="partition"))
            if cp > 8:
                for r in (1, 4):
                    rows.append(_case(EIGEN_ALIGNED, cp, r, single, p_for(EIGEN_ALIGNED, cp, r, "aligned")))
            else:
                for fam in (STAGED, STAGED_VIRTUAL):
                    for r in ((1, 2, 4) if cp == 4 else (1, 4)):
                        if 32 // cp * r >= 4:
                            rows.append(_case(fam, cp, r, single, p_for(fam, cp, r, "aligned"),
                                              tips=24 if fam == STAGED_VIRTUAL else 20))
    # aligned lists whose Ppad is not a multiple of G * R: the predicated kernel at (CP 1, R 4) and (CP 2, R 4)
    rows += [_case(EIGEN_PREDICATED, 1, 4, False, 301), _case(EIGEN_PREDICATED, 2, 4, False, 96),
             _case(EIGEN_PREDICATED, 1, 4, True, 96), _case(EIGEN_PREDICATED, 2, 4, True, 1)]
    # one live pattern: every other lane and r slot of the warp idle
    rows += [_case(MATRIX, 4, 2, False, 1), _case(MATRIX, 1, 4, True, 1),
             _case(EIGEN_PREDICATED, 32, 1, False, 1, lists="partition"), _case(EIGEN_ALIGNED, 16, 1, False, 1),
             _case(STAGED, 4, 1, True, 1), _case(STAGED_VIRTUAL, 1, 1, False, 1)]
    # every category lane live
    rows += [_case(STAGED, 4, 4, False, 301, C=4), _case(STAGED_VIRTUAL, 8, 1, False, 96, C=8),
             _case(EIGEN_PREDICATED, 8, 4, True, 1000, C=8, lists="partition"), _case(MATRIX, 8, 2, False, 33, C=8)]
    # fewer than four states on the 4-state kernels: tip states >= S are gaps
    rows += [_case(STAGED, 4, 4, False, 301, S=2), _case(STAGED_VIRTUAL, 8, 4, True, 1000, S=3),
             _case(EIGEN_PREDICATED, 4, 2, False, 96, S=3, lists="partition"), _case(MATRIX, 2, 1, False, 33, S=3),
             _case(EIGEN_ALIGNED, 16, 4, False, 96, S=2)]
    # scaling on every family and CP at R = 4, raw and SCALERS_LOG alternating, in-list cumulative index on some
    out = []
    for i, c in enumerate(rows):
        if c.r == 4:
            c = c._replace(scale="write" if c.family == STAGED_VIRTUAL or i % 3 == 0 else "cum", log=i % 2 == 1)
        out.append(c)
    # no knobs: 200 x 5000 at C = 4 keeps walkR 4 (157 warps of 32 patterns per subtree >= 132 SMs) and its wide phases
    # run the staged walk with virtual cherries; 64 x 2000 at C = 24 (CP 32) runs EigenAligned at R = 4
    out += [_case(STAGED_VIRTUAL, 4, 4, False, 5000, C=4, tips=200, natural=True, env={}),
            _case(EIGEN_ALIGNED, 32, 4, False, 2000, C=24, tips=64, natural=True, env={})]
    return out


CASES = _cases()


def _id(c):
    return (f"{FAMILY[c.family]}-cp{c.cp}-r{c.r}-{'f32' if c.single else 'f64'}-C{c.C}-S{c.S}-P{c.P}-{c.lists}"
            f"{'-set' if c.matrices == 'set' else ''}{'-' + c.scale if c.scale else ''}{'-log' if c.log else ''}"
            f"{'-natural' if c.natural else ''}")


# ---- the engine side of a case ------------------------------------------------------------------------------------------
PHASE = re.compile(r"\[b200-beagle\] phase (\d+): (\d+) walks over (\d+) patterns, kernel (\d+), R (\d+), (thin|wide)")
VIRTUAL = re.compile(r"\[b200-beagle\] plan: \d+ ops \((\d+) virtual cherries\)")
WALKR = re.compile(r"\[b200-beagle\] plan: .*, walkR (\d+)")


def _phases(err):
    return [tuple(int(x) for x in m.groups()[1:5]) + (m.group(6) == "thin",) for m in PHASE.finditer(err)]


class WalkTwin(Twin):
    """Twin with the post-order lists of this file.  Parity-1 destinations: internal node n at N + n (Twin's pre-order
    slots); spare buffers 2N .. 2N + 3.  Post-order factors of node n at n - T, the cumulative buffer at 2N."""

    def __init__(self, case, seed):
        self.case = case
        env = dict(case.env, B200_BEAGLE_DEBUG="1")
        pref = (SINGLE if case.single else 0) | (SCALERS_LOG if case.log else 0)
        super().__init__(case.S, case.C, case.tips, case.P, seed, pref=pref, env=env, nDiff=0,
                         partialTips=0.05 if case.family == STAGED_VIRTUAL else 0.25)
        if case.single:
            assert self.gpu.getDetails().flags & SINGLE
        self.rng = np.random.default_rng(seed + 7)
        self.lengths = np.asarray([self.tree.branchLength(n) for n in self.edges])
        self.parts = _parts(self.P) if case.lists == "partition" else [self.P]
        if case.lists == "partition":
            self.both("setPatternPartitions", len(self.parts), I32(np.repeat(np.arange(len(self.parts)), self.parts)))
        self.internal = list(range(self.T, self.N))
        self.cum_in_list = NONE                     # the cumulative index by-partition ops carry
        self.k = {}                                 # k_n: stored buffers in n's subtree
        for n in range(self.N):
            if n < self.T:
                self.k[n] = int(n in self.partialTips)
            else:
                c1, c2 = (int(c) for c in self.tree.child[n])
                self.k[n] = 1 + self.k[c1] + self.k[c2]
        self.subtree = {}
        for n in range(self.N):
            self.subtree[n] = [n] + ([] if n < self.T else [m for c in self.tree.child[n] for m in self.subtree[int(c)]])
        self.spares = [self.N + n for n in self.internal] + [2 * self.N + q for q in range(4)]

    # ---- inputs -------------------------------------------------------------------------------------------------------
    def new_lengths(self):
        self.lengths = self.lengths * self.rng.uniform(0.8, 1.25, len(self.edges))
        if self.case.matrices == "set":             # no eigen system behind these: the matrix-form walk
            for n, t in zip(self.edges, self.lengths):
                self.both("setTransitionMatrix", n, self.ora._transition(0, t, self.r[0]).reshape(-1), 0.0)
        else:
            self.both("updateTransitionMatrices", 0, I32(self.edges), None, None, self.lengths, len(self.edges))

    def new_eigen_system(self):
        S = self.S
        model = em.GTR(2.0, 3.0, 0.5, 1.5, 4.0, 1.0, np.array([0.25, 0.27, 0.23, 0.25])) if S == 4 else \
            em.SubstitutionModel(self.rng.uniform(0.2, 3.0, S * (S - 1) // 2), self.rng.dirichlet(np.full(S, 5.0)))
        ed = model.getEigenDecomposition()
        self.both("setEigenDecomposition", 0, ed.Evec.reshape(-1), ed.Ievc.reshape(-1), ed.Eval)
        self.both("setStateFrequencies", 0, model.getFrequencies())

    def fill_spares(self):
        P, S, C = self.P, self.S, self.C
        for b in self.spares:
            self.both("setPartials", b, self.rng.uniform(0.05, 1.0, P * S * C))
        return {b: self.partials(self.gpu, b) for b in self.spares}

    # ---- lists ----------------------------------------------------------------------------------------------------------
    def ops(self, parity=0, sw=None, sr=None, parts=None):
        """internal nodes children first; sw(n) / sr(n): the op's scale write / read buffer or NONE"""
        dest = (lambda n: n) if parity == 0 else (lambda n: n if n < self.T else self.N + n)
        flat, by_part = [], self.case.lists == "partition"
        for part in (parts if parts is not None else range(len(self.parts))) if by_part else [None]:
            for n in self.internal:
                c1, c2 = (int(c) for c in self.tree.child[n])
                op = [dest(n), sw(n) if sw else NONE, sr(n) if sr else NONE, dest(c1), c1, dest(c2), c2]
                flat += op + ([part, self.cum_in_list] if by_part else [])
        return flat

    def run(self, flat, cum=NONE):
        by_part = self.case.lists == "partition"
        count = len(flat) // (9 if by_part else 7)
        if by_part:
            self.both("updatePartialsByPartition", I32(flat), count)
        else:
            self.both("updatePartials", I32(flat), count, cum)

    def root_values(self, cum=NONE):
        out = []
        for b in (self.gpu, self.ora):
            v, site = np.zeros(1), np.zeros(self.P)
            b.calculateRootLogLikelihoods(I32([self.root]), I32([0]), I32([0]), I32([cum]), 1, v)
            b.getSiteLogLikelihoods(site)
            out.append((float(v[0]), site))
        return out

    # ---- checks -------------------------------------------------------------------------------------------------------
    def site_bound(self):
        return 1.001 * self.k[self.root] * U + 1e-9

    def check_root(self, cum=NONE):
        (lg, sg), (lo, so) = self.root_values(cum)
        if self.case.single:
            assert np.all(np.abs(sg - so) <= self.site_bound()), np.max(np.abs(sg - so))
            assert abs(lg - lo) <= float(np.sum(self.weights)) * self.site_bound()
        else:
            assert abs(lg - lo) <= 1e-10 * abs(lo), (lg, lo)
            assert np.allclose(sg, so, rtol=1e-10, atol=1e-12), np.max(np.abs(sg - so))

    def logf(self, b, idx):
        out = np.zeros(self.P)
        b.getLogScaleFactors(idx, out)
        return out

    def check_partials(self, parity=0, factor=None):
        """every internal buffer, whole; factor(n): the scale buffer of node n's op (None: unscaled).  fp32 with factors
        compares the unscaled values: stored value times exp(sum of its subtree's log factors)"""
        buf = (lambda n: n) if parity == 0 else (lambda n: self.N + n)
        C, P, S = self.C, self.P, self.S
        for n in self.internal:
            g, o = self.partials(self.gpu, buf(n)), self.partials(self.ora, buf(n))
            assert np.all(np.isfinite(g)), n
            if not self.case.single:
                assert _close(g, o), (n, np.max(np.abs(g - o) / (np.abs(o) + 1e-300)))
                continue
            assert o.min() > 2.0 ** -120, (n, o.min())          # fp32 normal range
            if factor is not None:
                lg = sum((self.logf(self.gpu, factor(m)) for m in self.subtree[n] if m >= self.T and factor(m) != NONE),
                         np.zeros(P))
                lo = sum((self.logf(self.ora, factor(m)) for m in self.subtree[n] if m >= self.T and factor(m) != NONE),
                         np.zeros(P))
                g = (g.reshape(C, P, S) * np.exp(lg)[None, :, None]).reshape(-1)
                o = (o.reshape(C, P, S) * np.exp(lo)[None, :, None]).reshape(-1)
            bound = 1.001 * self.k[n] * U + 1e-9
            assert np.all(np.abs(g - o) <= bound * o), (n, np.max(np.abs(g - o) / o) / bound)

    def check_factors(self, written, cum=NONE):
        """every written factor buffer and the cumulative buffer, as log factors"""
        for n in written:
            a, b = self.logf(self.gpu, n - self.T), self.logf(self.ora, n - self.T)
            if self.case.single:
                assert np.all(np.abs(a - b) <= 2.002 * self.k[n] * U + 1e-9), n
            else:
                assert np.allclose(a, b, rtol=1e-10, atol=1e-12), n
        assert np.any(self.logf(self.ora, written[0] - self.T) != 0.0)
        if cum != NONE:
            a, b = self.logf(self.gpu, cum), self.logf(self.ora, cum)
            if self.case.single:
                assert np.all(np.abs(a - b) <= self.site_bound())
            else:
                assert np.allclose(a, b, rtol=1e-10, atol=1e-12)

    def check_untouched(self, before, buffers):
        for b in buffers:
            assert np.array_equal(self.partials(self.gpu, b), before[b]), b


def _route_ok(case, err, sms):
    """the targeted cell ran; rows without knobs: the instance's walkR is the one the row states, and every phase is what
    b200DebugWalkRoute gives for its parameters"""
    phases, virtual = _phases(err), sum(int(v) for v in VIRTUAL.findall(err))
    assert phases, "no walk phase was launched"
    assert (case.family, case.r) in {(k, r) for _, _, k, r, _ in phases}, phases
    if case.family == STAGED_VIRTUAL:
        assert virtual > 0
    if case.natural:
        walk_r = {int(w) for w in WALKR.findall(err)}
        assert walk_r == {case.r}, walk_r
        lib = beagle.load_library()
        for n_subs, window, kernel, r, thin in phases:
            out = np.zeros(3, dtype=np.int32)
            assert lib.b200DebugWalkRoute(case.cp, _ppad(case.P), sms, case.r, 1, int(case.single), n_subs, window, 1, 1,
                                          int(virtual > 0), out.ctypes.data_as(beagle._IP)) == 0
            assert (kernel, r, thin) == (int(out[0]), int(out[1]), bool(out[2])), (n_subs, window)
    return len(phases) + (virtual > 0)                   # launches: the phases and the cherry snapshot


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_walk_route(case, sms, capfd):
    """Route: the cell (family, CP, R, precision) the row names, reached by the inputs of its row (module docstring):
    walk4Route in walk4e.cu, called by api.cu launchPlan once per phase.  Checks, node by node against the oracle: a
    fresh plan, a cache hit, a captured graph and its replay, the in-place eigen patch of that graph; untouched buffers;
    one-partition updates; rescaled lists and lists that read factors back."""
    capfd.readouterr()
    tw = WalkTwin(case, seed=1000 + CASES.index(case))
    try:
        before = tw.fill_spares()
        flat = tw.ops()
        # 1. a fresh plan, a cache hit, a graph capture that replays; then a new eigen system: the captured launches patched
        for step in range(4):
            if step == 3:
                tw.new_eigen_system()
            tw.new_lengths()
            tw.run(flat)
            err = capfd.readouterr().err
            if step == 0:
                launches = _route_ok(case, err, sms)
            else:                                        # cache hits: planned once
                assert "[b200-beagle] plan:" not in err, err
            if step == 2 and launches >= 2:
                assert "[b200-beagle] graph captured" in err, err
            if step == 3 and launches >= 2:             # the graph replayed (patched in place), nothing launched anew
                assert not _phases(err) and "graph capture" not in err, err
            tw.check_root()
            tw.check_partials()
        tw.check_untouched(before, tw.spares)
        # 2. one partition alone: the other partitions' columns of every destination keep their values
        if case.lists == "partition" and len(tw.parts) > 1:
            tw.new_lengths()
            tw.run(tw.ops(parts=[1]))
            tw.check_partials()
            tw.check_untouched(before, tw.spares)
        if case.scale is None:
            return
        # 3. rescaled: every other op with an internal child writes its factor (never a cherry); in-list cumulative index
        # or the factors accumulated after the list
        scaled = [n for q, n in enumerate(tw.internal)
                  if q % 2 == 1 and any(int(c) >= tw.T for c in tw.tree.child[n])]
        sw = lambda n: n - tw.T if n in scaled else NONE
        cum = tw.cumPost
        tw.both("resetScaleFactors", cum)
        tw.new_lengths()
        if case.scale == "cum":
            tw.cum_in_list = cum
            tw.run(tw.ops(sw=sw), cum)
        else:
            tw.run(tw.ops(sw=sw))
            tw.both("accumulateScaleFactors", I32([n - tw.T for n in scaled]), len(scaled), cum)
        err = capfd.readouterr().err
        if case.family == STAGED_VIRTUAL:
            assert sum(int(v) for v in VIRTUAL.findall(err)) > 0, err
        assert (case.family, case.r) in {(k, r) for _, _, k, r, _ in _phases(err)}, err
        tw.check_partials(factor=sw)
        tw.check_factors(scaled, cum)
        tw.check_root(cum)
        tw.check_untouched(before, tw.spares)
        # 4. parity-1 destinations; the ops that wrote a factor above read it back through destinationScaleRead
        tw.cum_in_list = NONE
        sr = lambda n: n - tw.T if n in scaled else NONE
        tw.run(tw.ops(parity=1, sr=sr))
        assert (case.family, case.r) in {(k, r) for _, _, k, r, _ in _phases(capfd.readouterr().err)}
        tw.check_partials(parity=1, factor=sr)
        tw.check_untouched(before, [2 * tw.N + q for q in range(4)])
    finally:
        tw.finalize()
