"""Joint ancestral-state sampling on the device (b200SampleAncestralStates, csrc/ancestral.cu).

Checked against the numpy restatement (oracle/ancestral.py) fed with the engine's own getPartials / getTransitionMatrix and
the same Philox uniforms: categories and states must be equal for every (row, pattern), except in a pattern where some draw's
uniform lies within 1e-12 of a CDF boundary (there a last-bit difference in a cumulative sum may pick the neighbour; those
patterns are counted and reported).  The sampled distribution is checked against exact enumeration."""
import ctypes as C
import os

import numpy as np
import pytest

from beast_mcmc_b200 import beagle
from harness import evomodel as em
from oracle import ancestral as anc

pytestmark = pytest.mark.gpu

NONE = -1
BOUNDARY = 1e-12
OUT_OF_RANGE = beagle.BeagleErrorCode.OUT_OF_RANGE_ERROR


def _random_tree(T, rng):
    """[(node, child1, child2)] in post-order; tips 0..T-1, internal nodes T..2T-2, root last."""
    nodes, ops = list(range(T)), []
    for nxt in range(T, 2 * T - 1):
        a, b = sorted(rng.choice(len(nodes), 2, replace=False), reverse=True)
        ca, cb = nodes.pop(a), nodes.pop(b)
        ops.append((nxt, cb, ca))
        nodes.append(nxt)
    return ops


def _model(S, seed):
    if S == 4:
        return em.GTR(1.0, 4.0, 0.7, 1.2, 5.0, 1.0, np.array([0.30, 0.22, 0.24, 0.24]))
    if S == 61:
        return em.MG94HKYCodonModel(1.0, 0.3, 2.0)
    rng = np.random.default_rng(seed)
    return em.SubstitutionModel(rng.uniform(0.2, 3.0, S * (S - 1) // 2), rng.dirichlet(np.full(S, 5.0)))


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


class Case:
    """A seeded instance driven through the C ABI: tips 0..T-1 (compact states with gaps, some given as ambiguity partials),
    internal nodes T..2T-2, matrix buffer = node index; rows = the nodes in pre-order."""

    def __init__(self, S=4, C=4, T=12, P=300, seed=3, partialTips=2, columns=None):
        rng = np.random.default_rng(seed)
        self.S, self.C, self.T, self.N = S, C, T, 2 * T - 1
        self.ops = _random_tree(T, rng)
        self.root = self.ops[-1][0]
        if columns is not None:
            self.states = np.asarray(columns, dtype=np.int32)
            P = self.states.shape[1]
        else:
            self.states = rng.integers(0, S + 1, size=(T, P)).astype(np.int32)            # S = gap
        self.P = P
        self.tipPartials = {}
        for t in range(T - partialTips, T):
            amb = (rng.random((P, S)) < 0.3).astype(np.float64)
            amb[np.arange(P), self.states[t] % S] = 1.0
            self.tipPartials[t] = amb
        self.lengths = rng.uniform(0.02, 0.3, self.N)
        self.model = _model(S, seed)
        site = em.GammaSiteRateModel(shape=0.5, gammaCategoryCount=C) if C > 1 else em.GammaSiteRateModel()
        self.rates, self.weights = site.getCategoryRates(), site.getCategoryProportions()
        kids = {n: (a, b) for n, a, b in self.ops}
        self.rows, stack = [], [(self.root, -1)]
        while stack:
            node, parent = stack.pop()
            self.rows.append((node, parent, node))
            for k in kids.get(node, ()):
                stack.append((k, len(self.rows) - 1))

    def arrays(self):
        nb, pr, mi = (np.array([r[k] for r in self.rows], dtype=np.int32) for k in range(3))
        return nb, pr, mi

    def create(self, resource=1, scaled=False, requirement=0):
        args = (self.T, self.N, self.T, self.S, self.P, 1, self.N, self.C, self.T if scaled else 0)
        inst = beagle.BeagleJNIImpl(*args, [resource, 0], 0, requirement)
        ed = self.model.getEigenDecomposition()
        inst.setEigenDecomposition(0, ed.Evec.ravel(), ed.Ievc.ravel(), ed.Eval)
        inst.setStateFrequencies(0, self.model.getFrequencies())
        inst.setCategoryWeights(0, self.weights)
        inst.setCategoryRates(self.rates)
        for t in range(self.T):
            if t in self.tipPartials:
                inst.setTipPartials(t, self.tipPartials[t].ravel())
            else:
                inst.setTipStates(t, self.states[t])
        self.scaled = scaled
        return inst

    def evaluate(self, inst, lengths=None):
        lengths = self.lengths if lengths is None else lengths
        idx = np.array([n for n in range(self.N) if n != self.root], dtype=np.int32)
        inst.updateTransitionMatrices(0, idx, None, None, lengths[idx], len(idx))
        flat = []
        for n, a, b in self.ops:
            sw = n - self.T if self.scaled else NONE
            flat += [n, sw, NONE, a, a, b, b]
        inst.updatePartials(np.array(flat, dtype=np.int32), len(self.ops), NONE)

    def sample(self, inst, seed=7, drawIndex=0):
        nb, pr, mi = self.arrays()
        return inst.sampleAncestralStates(nb, pr, mi, self.root, 0, 0, seed, drawIndex)

    def oracle_draws(self, inst, seed=7, drawIndex=0):
        """the restatement fed with the engine's own partials and matrices"""
        partials, mats = {}, {}
        for node, _, m in self.rows:
            if node >= self.T or node in self.tipPartials:
                out = np.zeros(self.C * self.P * self.S)
                inst.getPartials(node, NONE, out)
                partials[node] = out.reshape(self.C, self.P, self.S)
            if node != self.root:
                out = np.zeros(self.C * self.S * self.S)
                inst.getTransitionMatrix(m, out)
                mats[m] = out.reshape(self.C, self.S, self.S)
        tips = {t: self.states[t] for t in range(self.T) if t not in self.tipPartials}
        return anc.sample(self.rows, self.root, partials, tips, mats, self.weights, self.model.getFrequencies(), seed, drawIndex)


def _assert_same_draws(got, want, label):
    (states, cats), (ostates, ocats, margins) = got, want
    near = (margins < BOUNDARY).any(axis=0)
    ok = ~near
    print(f"{label}: {int(near.sum())} of {near.size} patterns hold a draw within {BOUNDARY:g} of a CDF boundary; "
          f"smallest margin {margins.min():.3e}")
    assert near.mean() <= 0.01, near.sum()
    assert np.array_equal(cats[ok], ocats[ok]), label
    bad = np.argwhere(states[:, ok] != ostates[:, ok])
    assert bad.size == 0, (label, bad[:5])


@pytest.mark.parametrize("S", [4, 20, 61])
@pytest.mark.parametrize("C", [1, 4])
def test_same_draws_as_restatement(S, C):
    T, P = (12, 300) if S == 4 else ((9, 160) if S == 20 else (7, 64))
    case = Case(S=S, C=C, T=T, P=P, seed=S + C)
    inst = case.create()
    case.evaluate(inst)
    got = case.sample(inst, seed=2024, drawIndex=5)
    assert got[0].shape == (case.N, P) and got[1].shape == (P,)
    assert ((got[0] >= 0) & (got[0] < S)).all() and ((got[1] >= 0) & (got[1] < C)).all()
    # compact tips keep their observed states
    for r, (node, _, _) in enumerate(case.rows):
        if node < case.T and node not in case.tipPartials:
            obs = case.states[node] < S
            assert np.array_equal(got[0][r][obs], case.states[node][obs])
    _assert_same_draws(got, case.oracle_draws(inst, seed=2024, drawIndex=5), f"S={S} C={C}")
    inst.finalize()


def test_single_precision_same_draws_as_restatement():
    case = Case(S=4, C=4, T=16, P=500, seed=41)
    inst = case.create(requirement=beagle.BeagleFlag.PRECISION_SINGLE)
    assert inst.getDetails().getFlags() & beagle.BeagleFlag.PRECISION_SINGLE
    case.evaluate(inst)
    _assert_same_draws(case.sample(inst, 11, 1), case.oracle_draws(inst, 11, 1), "single")
    inst.finalize()


def test_distribution_matches_exact_enumeration():
    """5 tips, one column repeated 200k times: one call = 200k independent joint draws (the counter carries the pattern)."""
    column = np.array([0, 1, 0, 2, 4], dtype=np.int32)           # tip 4 is a gap
    N = 200_000
    case = Case(S=4, C=2, T=5, seed=8, partialTips=0, columns=np.repeat(column[:, None], N, axis=1))
    inst = case.create()
    case.evaluate(inst)
    states, cats = case.sample(inst, seed=99, drawIndex=0)
    mats = {}
    for node, _, m in case.rows[1:]:
        out = np.zeros(case.C * 16)
        inst.getTransitionMatrix(m, out)
        mats[m] = out.reshape(case.C, 4, 4)
    parents = [r[1] for r in case.rows]
    mrows = [None] + [mats[r[2]] for r in case.rows[1:]]
    tipL = {r: (np.ones(4) if column[node] >= 4 else np.eye(4)[column[node]])
            for r, (node, _, _) in enumerate(case.rows) if node < case.T}
    outcomes, probs = anc.enumerate_joint(parents, mrows, tipL, case.weights, case.model.getFrequencies())
    internal = [r for r in range(len(case.rows)) if r not in tipL]
    keys = cats.astype(np.int64)
    for r in internal:
        keys = keys * 4 + states[r]
    counts = np.bincount(keys, minlength=len(outcomes)) / N
    want = np.zeros(len(outcomes))
    for o, pr in zip(outcomes, probs):
        k = o[0]
        for x in o[1:]:
            k = k * 4 + x
        want[k] = pr
    # every outcome within 5 binomial standard deviations plus 3 counts
    bound = 5 * np.sqrt(want * (1 - want) / N) + 3.0 / N
    worst = np.max(np.abs(counts - want) / bound)
    print(f"distribution: {len(outcomes)} outcomes, largest deviation {worst:.3f} of the bound")
    assert worst <= 1.0
    inst.finalize()


def test_rescaled_instance_draws_as_unscaled():
    case = Case(S=4, C=4, T=40, P=400, seed=12)
    plain = case.create()
    case.evaluate(plain)
    ref = case.sample(plain, 5, 3)
    margins = case.oracle_draws(plain, 5, 3)[2]
    scaled = case.create(scaled=True)
    case.evaluate(scaled)
    got = case.sample(scaled, 5, 3)
    ok = ~(margins < BOUNDARY).any(axis=0)
    assert np.array_equal(got[1][ok], ref[1][ok]) and np.array_equal(got[0][:, ok], ref[0][:, ok])
    plain.finalize(); scaled.finalize()


def test_virtual_cherries_on_off_bit_equal():
    case = Case(S=4, C=4, T=64, P=700, seed=13, partialTips=0)

    def run():
        inst = case.create()
        case.evaluate(inst)
        out = case.sample(inst, 17, 9)
        inst.finalize()
        return out

    on = run()
    off = _with_env({"B200_VIRTUAL_CHERRIES": "0"}, run)
    assert np.array_equal(on[0], off[0]) and np.array_equal(on[1], off[1])


def test_sampling_after_deferred_evaluation_sees_flushed_partials():
    case = Case(S=4, C=4, T=64, P=700, seed=14, partialTips=0)
    inst = case.create()
    case.evaluate(inst)
    out = np.zeros(1)
    inst.calculateRootLogLikelihoods(np.array([case.root], np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32),
                                     np.array([NONE], np.int32), 1, out)
    # move one branch: a short matrix update and the root path, both deferred (csrc/incr.cu), then sample at once
    lengths = case.lengths.copy()
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
    got = case.sample(inst, 3, 4)
    # a fresh instance evaluated at the moved lengths holds the partials the sample must have seen
    fresh = case.create()
    case.evaluate(fresh, lengths)
    a, b = np.zeros(case.C * case.P * 4), np.zeros(case.C * case.P * 4)
    inst.getPartials(case.root, NONE, a)
    fresh.getPartials(case.root, NONE, b)
    assert np.allclose(a, b, rtol=1e-12, atol=0)
    _assert_same_draws(got, case.oracle_draws(inst, 3, 4), "after deferred evaluation")
    inst.finalize(); fresh.finalize()


def test_same_draw_index_repeats_other_index_differs():
    case = Case(S=4, C=4, T=20, P=300, seed=15)
    inst = case.create()
    case.evaluate(inst)
    a, b, c = case.sample(inst, 1, 0), case.sample(inst, 1, 0), case.sample(inst, 1, 1)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert not np.array_equal(a[0], c[0])
    assert not np.array_equal(a[0], case.sample(inst, 2, 0)[0])
    inst.finalize()


def _shard_resource(devices):
    import torch
    n = torch.cuda.device_count()
    devices = [d % n for d in devices]
    res = [r.number for r in beagle.BeagleFactory.getResourceDetails() if "pattern-sharded" in r.name]
    assert res
    arr = (C.c_int * len(devices))(*devices)
    assert beagle.load_library().b200SetShardDevices(arr, len(devices)) == 0
    return res[0]


@pytest.mark.parametrize("S,P,g", [(4, 301, 3), (4, 2, 3), (20, 97, 2)])
def test_sharded_instance_bit_equal_to_single_device(S, P, g):
    case = Case(S=S, C=2, T=10, P=P, seed=16 + P)
    res = _shard_resource(list(range(g)))
    whole, sharded = case.create(), case.create(resource=res)
    assert sharded.getDetails().getResourceNumber() == res
    for inst in (whole, sharded):
        case.evaluate(inst)
    a, b = case.sample(whole, 21, 2), case.sample(sharded, 21, 2)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    whole.finalize(); sharded.finalize()


def test_errors_return_out_of_range_and_launch_nothing():
    case = Case(S=4, C=4, T=20, P=300, seed=17, partialTips=0)
    inst = case.create()
    lib = beagle.load_library()
    nb, pr, mi = case.arrays()
    R = len(nb)
    states = np.zeros((R, case.P), np.int32)
    cats = np.zeros(case.P, np.int32)

    def call(nb=nb, pr=pr, mi=mi, root=case.root, w=0, f=0):
        ip = lambda a: np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int))
        return lib.b200SampleAncestralStates(inst.instance, ip(nb), ip(pr), ip(mi), len(nb), root, w, f, 1, 0,
                                             ip(states), ip(cats))

    # internal buffers never written yet
    assert call() == OUT_OF_RANGE
    case.evaluate(inst)
    out = np.zeros(1)
    inst.calculateRootLogLikelihoods(np.array([case.root], np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32),
                                     np.array([NONE], np.int32), 1, out)
    # deferred work pending: a refused call must leave it pending (nothing launched), the root call then fuses it
    node = case.ops[2][0]
    inst.updateTransitionMatrices(0, np.array([node], np.int32), None, None, case.lengths[[node]] * 1.3, 1)
    fused = lib.b200GetFusedLaunches(inst.instance)
    swapped = pr.copy()
    child = int(np.nonzero(pr > 0)[0][0])
    swapped[child] = child                                          # a row as its own parent
    later = pr.copy()
    later[child] = R - 1                                            # parent after the child
    bad = [dict(pr=swapped), dict(pr=later), dict(nb=np.where(np.arange(R) == 3, 10_000, nb)),
           dict(mi=np.where(np.arange(R) == 3, -2, mi)), dict(root=-1), dict(root=10_000), dict(w=1), dict(f=-1),
           dict(pr=np.where(np.arange(R) == 0, 0, pr))]
    for kw in bad:
        states[:] = -7
        assert call(**kw) == OUT_OF_RANGE, kw
        assert (states == -7).all()
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
    assert call() == 0
    inst.finalize()
