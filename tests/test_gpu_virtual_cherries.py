"""Virtual cherries (walk4e.cu, api.cu): a tip x tip op without rescaling is not run; the eigen-form walk recomputes it where
it reads it, and every other reader gets its partials written first.  Everything must be bit-identical to storing the
cherries (B200_VIRTUAL_CHERRIES=0), and equal the oracle driven by the same call sequence."""
import os
import re

import numpy as np
import pytest

from beast_mcmc_b200 import beagle
from harness import evomodel as em
from oracle.felsenstein import OracleBeagle

pytestmark = pytest.mark.gpu

NONE = -1
REL = 1e-10


def _random_tree(T, rng):
    """[(node, child1, child2)] in post-order; tips 0..T-1, internal nodes T..2T-2, root last."""
    nodes, ops = list(range(T)), []
    for nxt in range(T, 2 * T - 1):
        a, b = sorted(rng.choice(len(nodes), 2, replace=False), reverse=True)
        ca, cb = nodes.pop(a), nodes.pop(b)
        ops.append((nxt, cb, ca))
        nodes.append(nxt)
    return ops


class Case:
    """A seeded 4-state instance driven through the C ABI.  Buffers: post(node, parity), pre(node); matrices: mat(node,
    parity)."""

    def __init__(self, T=64, P=1000, C=4, seed=5):
        rng = np.random.default_rng(seed)
        self.T, self.P, self.C, self.N = T, P, C, 2 * T - 1
        self.ops = _random_tree(T, rng)
        self.root = self.ops[-1][0]
        self.parent = {c: n for n, a, b in self.ops for c in (a, b)}
        self.cherries = [(n, a, b) for n, a, b in self.ops if a < T and b < T]
        self.states = rng.integers(0, 5, size=(T, P)).astype(np.int32)          # 4 = gap
        self.lengths = rng.uniform(0.01, 0.3, self.N)
        self.model = em.GTR(1.0, 4.0, 0.7, 1.2, 5.0, 1.0, np.array([0.30, 0.22, 0.24, 0.24]))
        site = em.GammaSiteRateModel(shape=0.5, gammaCategoryCount=C) if C > 1 else em.GammaSiteRateModel()
        self.rates, self.weights = site.getCategoryRates(), site.getCategoryProportions()
        self.patternWeights = rng.integers(1, 5, P).astype(np.float64)

    def post(self, node, par=0):
        return node if node < self.T or par == 0 else self.N + node - self.T

    def pre(self, node):
        return 2 * self.N - self.T + node

    def mat(self, node, par=0):
        return node + par * self.N

    def create(self, gpu):
        args = (self.T, 2 * self.N - self.T + self.N, self.T, 4, self.P, 1, 2 * self.N, self.C, 0)
        inst = beagle.BeagleJNIImpl(*args, [1, 0], 0, 0) if gpu else OracleBeagle(*args)
        ed = self.model.getEigenDecomposition()
        inst.setEigenDecomposition(0, ed.Evec.ravel(), ed.Ievc.ravel(), ed.Eval)
        inst.setStateFrequencies(0, self.model.getFrequencies())
        inst.setCategoryWeights(0, self.weights)
        inst.setCategoryRates(self.rates)
        inst.setPatternWeights(self.patternWeights)
        for t in range(self.T):
            inst.setTipStates(t, self.states[t])
        return inst

    def matrices(self, inst, nodes, par=0, lengths=None):
        lengths = self.lengths if lengths is None else lengths
        idx = np.array([self.mat(n, par) for n in nodes], dtype=np.int32)
        inst.updateTransitionMatrices(0, idx, None, None, np.array([lengths[n] for n in nodes]), len(nodes))

    def update(self, inst, ops, par=0):
        flat = []
        for n, a, b in ops:
            flat += [self.post(n, par), NONE, NONE, self.post(a, par), self.mat(a, par), self.post(b, par), self.mat(b, par)]
        inst.updatePartials(np.array(flat, dtype=np.int32), len(ops), NONE)

    def root_value(self, inst, par=0):
        out = np.zeros(1)
        inst.calculateRootLogLikelihoods(np.array([self.post(self.root, par)], dtype=np.int32), np.zeros(1, np.int32),
                                         np.zeros(1, np.int32), np.array([NONE], np.int32), 1, out)
        return out[0]

    def partials(self, inst, buf):
        out = np.zeros(self.C * self.P * 4)
        inst.getPartials(buf, NONE, out)
        return out

    def path(self, node):
        """ops from node's parent up to the root"""
        out, n = [], node
        by_node = {o[0]: o for o in self.ops}
        while n != self.root:
            n = self.parent[n]
            out.append(by_node[n])
        return out


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


def _virtual_count(text):
    return sum(int(m) for m in re.findall(r"\((\d+) virtual cherries\)", text))


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


@pytest.mark.parametrize("C,P,first", [(4, 1000, "preorder"), (1, 1000, "preorder"), (4, 5000, "preorder"),
                                        (4, 1000, "edge"), (4, 1000, "cross")])
def test_full_evaluation_bit_equal_to_stored_cherries(C, P, first, capfd):
    """Joint value, every post-order buffer, pre-order partials, edge and cross-product derivatives of a full evaluation:
    switch on == switch off, bit for bit.  `first` is the reader that meets the unstored cherries (getPartials comes
    last, after every cherry has been stored)."""
    case = Case(T=64, P=P, C=C, seed=7)
    internal = [n for n, _, _ in case.ops]
    non_root = [n for n in range(case.N) if n != case.root]
    post = np.array([case.post(n) for n in non_root], np.int32)
    pre = np.array([case.pre(n) for n in non_root], np.int32)

    def preorder(inst, out):
        # root pre-partials = frequencies; parents before children
        inst.setPartials(case.pre(case.root), np.tile(case.model.getFrequencies(), case.C * case.P))
        pre_ops = []
        for n, a, b in reversed(case.ops):
            for child, sib in ((a, b), (b, a)):
                pre_ops += [case.pre(child), NONE, NONE, case.pre(n), case.mat(child), case.post(sib), case.mat(sib)]
        inst.updatePrePartials(np.array(pre_ops, dtype=np.int32), len(pre_ops) // 7, NONE)

    def edge(inst, out):
        per = np.zeros(len(non_root) * case.P)
        s1, s2 = np.zeros(len(non_root)), np.zeros(len(non_root))
        inst.calculateEdgeDifferentials(post, pre, np.array([case.mat(n) for n in non_root], np.int32),
                                        np.zeros(1, np.int32), len(non_root), per, s1, s2)
        out["derivatives"], out["sum"], out["sumsq"] = per, s1, s2

    def cross(inst, out):
        acc = np.zeros(16)
        inst.calculateCrossProductDifferentials(post, pre, np.zeros(1, np.int32), np.zeros(1, np.int32),
                                                np.array([case.lengths[n] for n in non_root]), len(non_root), acc, None)
        out["cross"] = acc

    def run():
        inst = case.create(True)
        case.matrices(inst, non_root)
        case.update(inst, case.ops)
        out = {"root": np.array([case.root_value(inst)])}
        if first == "preorder":
            preorder(inst, out)
        else:        # pre-order partials from elsewhere: the derivative call is the first reader of the post buffers
            rng = np.random.default_rng(5)
            for n in non_root:
                inst.setPartials(case.pre(n), rng.uniform(0.1, 1.0, case.C * case.P * 4))
        {"preorder": edge, "edge": edge, "cross": cross}[first](inst, out)
        for n in non_root:
            out[f"pre{n}"] = case.partials(inst, case.pre(n))
        for n in internal:
            out[f"post{n}"] = case.partials(inst, case.post(n))
        inst.finalize()
        return out

    on = _with_env({"B200_VIRTUAL_CHERRIES": "1", "B200_BEAGLE_DEBUG": "1"}, run)
    assert _virtual_count(capfd.readouterr().err) == len(case.cherries) > 0
    off = _with_env({"B200_VIRTUAL_CHERRIES": "0", "B200_BEAGLE_DEBUG": "1"}, run)
    assert _virtual_count(capfd.readouterr().err) == 0
    for k in off:
        assert np.array_equal(on[k], off[k]), k


@pytest.mark.parametrize("fuse", ["0", "1"])
def test_cherry_keeps_its_matrices_after_they_are_overwritten(fuse, capfd):
    """A later list reads a cherry whose matrix buffer has been overwritten since: the cherry keeps the value it was
    computed with (as stored partials would), read by the walk (no fusion) or by the fused incremental evaluation."""
    case = Case(T=64, P=1000, C=4, seed=9)
    cherry, tip, _ = case.cherries[0]
    non_root = [n for n in range(case.N) if n != case.root]
    moved = case.lengths.copy()
    moved[tip] *= 3.0

    def run(inst):
        case.matrices(inst, non_root)
        case.update(inst, case.ops)
        first = case.root_value(inst)
        case.matrices(inst, [tip], lengths=moved)                       # one of the cherry's matrices, overwritten
        case.update(inst, case.path(cherry))                            # reads the cherry as a child
        return first, case.root_value(inst)

    gpu = {}
    for switch in ("1", "0"):
        env = {"B200_VIRTUAL_CHERRIES": switch, "B200_FUSE": fuse, "B200_BEAGLE_DEBUG": "1"}
        inst = _with_env(env, lambda: case.create(True))
        gpu[switch] = _with_env(env, lambda: run(inst))
        inst.finalize()
        if switch == "1":
            assert _virtual_count(capfd.readouterr().err) > 0
    oracle = case.create(False)
    want = run(oracle)
    assert gpu["1"] == gpu["0"]
    assert _rel(gpu["1"][1], want[1]) <= REL and _rel(gpu["1"][0], want[0]) <= REL


@pytest.mark.parametrize("fuse", ["0", "1"])
def test_list_reads_a_cherry_then_overwrites_it(fuse, capfd):
    """A list that reads a virtual cherry and later rewrites the same buffer (it runs in the caller's order): the read
    sees the cherry from the earlier list, through the walk (no fusion) or the fused incremental evaluation."""
    case = Case(T=64, P=1000, C=4, seed=23)
    cherry, tip, _ = case.cherries[0]
    non_root = [n for n in range(case.N) if n != case.root]
    by_node = {o[0]: o for o in case.ops}
    moved = case.lengths.copy()
    moved[tip] *= 2.0
    parent = case.parent[cherry]
    # the cherry's parent (reads the cherry), the cherry again (new matrix), then the parent's path to the root
    ops = [by_node[parent], by_node[cherry]] + case.path(parent)

    def run(inst):
        case.matrices(inst, non_root)
        case.update(inst, case.ops)
        first = case.root_value(inst)
        case.matrices(inst, [tip], lengths=moved)
        case.update(inst, ops)
        return first, case.root_value(inst), case.partials(inst, case.post(cherry))

    gpu = {}
    for switch in ("1", "0"):
        env = {"B200_VIRTUAL_CHERRIES": switch, "B200_FUSE": fuse, "B200_BEAGLE_DEBUG": "1"}
        inst = _with_env(env, lambda: case.create(True))
        gpu[switch] = _with_env(env, lambda: run(inst))
        inst.finalize()
        if switch == "1":
            assert _virtual_count(capfd.readouterr().err) > 0
    want = run(case.create(False))
    assert gpu["1"][:2] == gpu["0"][:2] and np.array_equal(gpu["1"][2], gpu["0"][2])
    assert _rel(gpu["1"][0], want[0]) <= REL and _rel(gpu["1"][1], want[1]) <= REL
    assert np.allclose(gpu["1"][2], want[2], rtol=1e-12, atol=0)


def test_set_tip_states_keeps_the_cherry_value():
    """setTipStates on a cherry's tip: the cherry keeps what it was computed from."""
    case = Case(T=64, P=1000, C=4, seed=13)
    cherry, tip, _ = case.cherries[0]
    non_root = [n for n in range(case.N) if n != case.root]
    new_states = np.random.default_rng(3).integers(0, 4, case.P).astype(np.int32)

    def run(switch, change):
        def go():
            inst = case.create(True)
            case.matrices(inst, non_root)
            case.update(inst, case.ops)
            case.root_value(inst)
            if change:
                inst.setTipStates(tip, new_states)
            out = case.partials(inst, case.post(cherry))
            inst.finalize()
            return out
        return _with_env({"B200_VIRTUAL_CHERRIES": switch}, go)

    stored = run("0", False)
    assert np.array_equal(run("1", True), stored)
    assert np.array_equal(run("0", True), stored)


@pytest.mark.parametrize("fuse", ["0", "1"])
def test_full_and_incremental_evaluations_interleaved(fuse, capfd):
    """Full evaluations in both buffer parities interleaved with incremental ones that rewrite a cherry: every step equals
    the oracle; after the first round no list is planned again (the plan cache keeps hitting), and once the full lists'
    graphs are captured (third use) nothing is captured again: they replay."""
    case = Case(T=64, P=1000, C=4, seed=17)
    cherry, tip, _ = case.cherries[0]
    non_root = [n for n in range(case.N) if n != case.root]
    rng = np.random.default_rng(1)
    steps = [case.lengths * rng.uniform(0.9, 1.1, case.N) for _ in range(12)]
    incremental = [next(o for o in case.ops if o[0] == cherry)] + case.path(cherry)

    def run(inst, record):
        vals = []
        for k, lengths in enumerate(steps):
            par = k % 2
            case.matrices(inst, non_root, par, lengths)
            case.update(inst, case.ops, par)
            vals.append(case.root_value(inst, par))
            moved = lengths.copy()
            moved[tip] *= 1.5
            case.matrices(inst, [tip], par, moved)
            case.update(inst, incremental, par)
            vals.append(case.root_value(inst, par))
            if record is not None:
                err = capfd.readouterr().err
                record.append((len(re.findall(r"\[b200-beagle\] plan:", err)),
                               len(re.findall(r"\[b200-beagle\] graph captured", err)),
                               len(re.findall(r"\[b200-beagle\] graph capture failed", err))))
        return vals

    env = {"B200_VIRTUAL_CHERRIES": "1", "B200_FUSE": fuse, "B200_BEAGLE_DEBUG": "1"}
    inst = _with_env(env, lambda: case.create(True))
    planned = []
    got = _with_env(env, lambda: run(inst, planned))
    inst.finalize()
    want = run(case.create(False), None)
    for g, w in zip(got, want):
        assert _rel(g, w) <= REL
    plans, captures, failures = (np.array([r[i] for r in planned]) for i in range(3))
    assert plans[:2].sum() > 0 and plans[2:].sum() == 0, planned
    assert captures[:6].sum() >= 2 and captures[6:].sum() == 0 and failures.sum() == 0, planned
