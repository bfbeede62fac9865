"""Sibling stack of the staged eigen walk (walk4e.cu, api.cu::assignStackSlots): a result that a later op of the same walk
reads back, other than through register forwarding, is also kept in a per-warp shared-memory slot and read from there.
Everything must be bit-identical to the route through global memory (B200_WALK_STACK_SLOTS=0), and equal the oracle."""
import os
import re

import numpy as np
import pytest

from beast_mcmc_b200 import beagle
from test_gpu_virtual_cherries import NONE, REL, Case, _rel, _with_env

pytestmark = pytest.mark.gpu

SINGLE = beagle.BeagleFlag.PRECISION_SINGLE


def _balanced_tree(T):
    """[(node, child1, child2)] of a complete binary tree over T = 2^k tips, post-order"""
    ops, nxt = [], T

    def build(lo, hi):
        nonlocal nxt
        if hi - lo == 1:
            return lo
        a, b = build(lo, (lo + hi) // 2), build((lo + hi) // 2, hi)
        ops.append((nxt, a, b))
        nxt += 1
        return nxt - 1
    build(0, T)
    return ops


class StackCase(Case):
    """Case with one scale buffer per node plus a cumulative one, and an optional PRECISION_SINGLE instance"""

    def __init__(self, T=256, P=2000, C=4, seed=5, balanced=False, single=False, rescale=False):
        super().__init__(T=T, P=P, C=C, seed=seed)
        if balanced:
            self.ops = _balanced_tree(T)
            self.root = self.ops[-1][0]
            self.parent = {c: n for n, a, b in self.ops for c in (a, b)}
        self.single, self.rescale = single, rescale

    def create(self, gpu):
        args = (self.T, 2 * self.N - self.T + self.N, self.T, 4, self.P, 1, 2 * self.N, self.C, self.N + 1)
        assert gpu
        inst = beagle.BeagleJNIImpl(*args, [1, 0], SINGLE if self.single else 0, 0)
        assert bool(inst.getDetails().flags & SINGLE) == self.single
        ed = self.model.getEigenDecomposition()
        inst.setEigenDecomposition(0, ed.Evec.ravel(), ed.Ievc.ravel(), ed.Eval)
        inst.setStateFrequencies(0, self.model.getFrequencies())
        inst.setCategoryWeights(0, self.weights)
        inst.setCategoryRates(self.rates)
        inst.setPatternWeights(self.patternWeights)
        for t in range(self.T):
            inst.setTipStates(t, self.states[t])
        return inst

    def update(self, inst, ops, par=0):
        if not self.rescale:
            return super().update(inst, ops, par)
        flat = []
        for n, a, b in ops:
            flat += [self.post(n, par), n, NONE, self.post(a, par), self.mat(a, par), self.post(b, par), self.mat(b, par)]
        inst.updatePartials(np.array(flat, dtype=np.int32), len(ops), NONE)

    def root_value(self, inst, par=0):
        cum = NONE
        if self.rescale:
            cum = self.N
            inst.resetScaleFactors(cum)
            idx = np.array([n for n, _, _ in self.ops], dtype=np.int32)
            inst.accumulateScaleFactors(idx, len(idx), cum)
        out = np.zeros(1)
        inst.calculateRootLogLikelihoods(np.array([self.post(self.root, par)], dtype=np.int32), np.zeros(1, np.int32),
                                         np.zeros(1, np.int32), np.array([cum], np.int32), 1, out)
        return out[0]

    def sites(self, inst):
        out = np.zeros(self.P)
        inst.getSiteLogLikelihoods(out)
        return out


def _counts(text):
    """(read from the stack, read from memory) summed over the plan lines"""
    rows = re.findall(r"(\d+) read from the stack, (\d+) from memory", text)
    return sum(int(a) for a, _ in rows), sum(int(b) for _, b in rows)


def _both(case, run, capfd, extra=None):
    """run() with the stack on (the default) and off: (on, off, (stack, memory) reads with the stack on)"""
    env = {"B200_BEAGLE_DEBUG": "1", **(extra or {})}
    assert "B200_WALK_STACK_SLOTS" not in os.environ
    on = _with_env(env, run)
    con = _counts(capfd.readouterr().err)
    off = _with_env({**env, "B200_WALK_STACK_SLOTS": "0"}, run)
    coff = _counts(capfd.readouterr().err)
    assert coff[0] == 0
    return on, off, con


def _full(case):
    def run():
        inst = case.create(True)
        case.matrices(inst, [n for n in range(case.N) if n != case.root])
        case.update(inst, case.ops)
        out = {"root": np.array([case.root_value(inst)]), "sites": case.sites(inst)}
        for n, _, _ in case.ops:
            out[f"post{n}"] = case.partials(inst, case.post(n))
        inst.finalize()
        return out
    return run


@pytest.mark.parametrize("kind", ["random", "rescaled", "single", "wide", "C1", "C8", "C8rescaled"])
def test_full_evaluation_bit_equal_to_memory_route(kind, capfd):
    """Root, site log-likelihoods and getPartials of every post-order buffer: stack on == stack off, bit for bit.
    rescaled: a scale write on every op; single: fp32 partials storage; wide: 10k patterns, so the phases run at R = 4.
    C1 / C8: other category counts, whose kernels are built without the stack: no slot is assigned there."""
    C = {"C1": 1, "C8": 8, "C8rescaled": 8}.get(kind, 4)
    case = StackCase(T=256, P=10000 if kind in ("wide", "C1") else 2000, C=C, seed=11, rescale="rescaled" in kind,
                     single=kind == "single")
    on, off, (stack, memory) = _both(case, _full(case), capfd)
    assert (stack > 0) == (C == 4)
    for k in off:
        assert np.array_equal(on[k], off[k]), k


def test_overflow_goes_through_memory(capfd):
    """One walk over a complete binary tree of 256 tips needs more live siblings than there are slots: the deepest ones
    travel through memory, and the results stay bit-identical."""
    case = StackCase(T=256, P=2000, seed=3, balanced=True)
    on, off, (stack, memory) = _both(case, _full(case), capfd, {"B200_PHASE_T": "100000"})
    assert stack > 0 and memory > 0          # one walk: every child read from memory is an overflowed sibling
    for k in off:
        assert np.array_equal(on[k], off[k]), k


@pytest.mark.parametrize("fuse", ["0", "1"])
def test_list_reads_a_buffer_then_rewrites_it(fuse, capfd):
    """A list that reads an internal buffer and later rewrites it (one walk in the caller's order): every read sees the
    value it should, with the stack on and off alike."""
    case = StackCase(T=64, P=1000, seed=23)
    by_node = {o[0]: o for o in case.ops}
    node = next(n for n, a, b in case.ops if a >= case.T and b >= case.T and n != case.root)
    parent = case.parent[node]
    moved = case.lengths * 1.7
    ops = [by_node[parent], by_node[node]] + case.path(node)     # reads node, rewrites it, then its path to the root

    def run():
        inst = case.create(True)
        case.matrices(inst, [n for n in range(case.N) if n != case.root])
        case.update(inst, case.ops)
        first = case.root_value(inst)
        case.matrices(inst, [by_node[node][1], by_node[node][2]], lengths=moved)
        case.update(inst, ops)
        out = (first, case.root_value(inst), case.partials(inst, case.post(node)), case.partials(inst, case.post(parent)))
        inst.finalize()
        return out

    on, off, _ = _both(case, run, capfd, {"B200_FUSE": fuse})
    assert on[:2] == off[:2] and np.array_equal(on[2], off[2]) and np.array_equal(on[3], off[3])


@pytest.mark.parametrize("fuse", ["0", "1"])
def test_incremental_evaluation_reads_stacked_siblings_from_memory(fuse, capfd):
    """After a full evaluation, a path update from a tip to the root reads the siblings along the path from global memory
    (walk or fused incremental launch): equal with the stack on and off, and equal to the oracle."""
    case = StackCase(T=256, P=2000, seed=29)
    tip = 0
    moved = case.lengths.copy()
    moved[tip] *= 2.5
    path = case.path(tip)

    def run(inst):
        case.matrices(inst, [n for n in range(case.N) if n != case.root])
        case.update(inst, case.ops)
        first = case.root_value(inst)
        case.matrices(inst, [tip], lengths=moved)
        case.update(inst, path)
        return first, case.root_value(inst)

    def gpu():
        inst = case.create(True)
        out = run(inst)
        inst.finalize()
        return out

    on, off, (stack, _) = _both(case, gpu, capfd, {"B200_FUSE": fuse})
    assert stack > 0 and on == off
    want = run(Case.create(case, False))
    assert _rel(on[0], want[0]) <= REL and _rel(on[1], want[1]) <= REL
