"""Joint ancestral-state sampling without a GPU: the numpy restatement (oracle/ancestral.py) against exact enumeration, its
Philox convention, and the host-side row rules of b200SampleAncestralStates (b200DebugAncestralRows, no CUDA calls)."""
import numpy as np

import helpers as H  # noqa: F401  (sets sys.path)
from beast_mcmc_b200 import beagle, build
from harness import evomodel as em
from oracle import ancestral as anc
from oracle.felsenstein import OracleBeagle

NONE = -1


def test_uniform_is_numpy_philox_first_word():
    # Philox4x64-10 at key (12345, 0), counter (7, 3, 2, 0): first output word 3063256571908658440 (the engine's
    # philox4x64_10 gives the same word; numpy reaches that block from counter - 1, including the borrow at drawIndex 0)
    assert anc.uniform(12345, 7, 3, 2) == (3063256571908658440 >> 11) * 2.0 ** -53
    assert anc.uniform(0, 0, 0, 0) == (1609277786247541068 >> 11) * 2.0 ** -53
    assert anc.uniform(12345, 7, 3, 2) != anc.uniform(12345, 8, 3, 2)


def test_draw_rule():
    assert anc.draw(np.array([0.2, 0.0, 0.8]), 0.1)[0] == 0
    assert anc.draw(np.array([0.2, 0.0, 0.8]), 0.2)[0] == 2          # a cumulative sum must EXCEED u * total
    assert anc.draw(np.array([0.0, 0.0, 0.0]), 0.5)[0] == 0           # impossible data: item 0
    j, margin = anc.draw(np.array([1.0, 1.0]), 0.5 + 1e-14)
    assert j == 1 and margin < 1e-12


def test_restatement_samples_exact_enumeration():
    """4 tips ((0,1),(2,3)) with one column repeated: the restatement's draws over patterns against the exact posterior."""
    S, Cn, P = 4, 2, 4000
    column = [0, 2, 4, 1]                                  # tip 2 is a gap
    model = em.HKY(4.0, np.array([0.3, 0.2, 0.2, 0.3]))
    site = em.GammaSiteRateModel(shape=0.5, gammaCategoryCount=Cn)
    w, rates = site.getCategoryProportions(), site.getCategoryRates()
    inst = OracleBeagle(4, 7, 4, S, P, 1, 7, Cn, 0)
    ed = model.getEigenDecomposition()
    inst.setEigenDecomposition(0, ed.Evec.ravel(), ed.Ievc.ravel(), ed.Eval)
    inst.setStateFrequencies(0, model.getFrequencies())
    inst.setCategoryWeights(0, w)
    inst.setCategoryRates(rates)
    for t in range(4):
        inst.setTipStates(t, np.full(P, column[t], dtype=np.int32))
    lengths = np.array([0.1, 0.3, 0.2, 0.05, 0.15, 0.25, 0.0])
    inst.updateTransitionMatrices(0, np.arange(6, dtype=np.int32), None, None, lengths[:6], 6)
    ops = [(4, 0, 1), (5, 2, 3), (6, 4, 5)]
    flat = []
    for n, a, b in ops:
        flat += [n, NONE, NONE, a, a, b, b]
    inst.updatePartials(np.array(flat, dtype=np.int32), 3, NONE)
    rows = [(6, -1, 6), (5, 0, 5), (3, 1, 3), (2, 1, 2), (4, 0, 4), (1, 4, 1), (0, 4, 0)]
    partials = {b: np.asarray(inst.partials[b]) for b in (4, 5, 6)}
    mats = {m: np.asarray(inst.matrices[m]) for m in range(6)}
    tips = {t: np.full(P, column[t]) for t in range(4)}
    states, cats, _ = anc.sample(rows, 6, partials, tips, mats, w, model.getFrequencies(), seed=5, drawIndex=0)
    assert (states[2] == 1).all() and (states[5] == 2).all() and (states[6] == 0).all()
    tipL = {r: (np.ones(S) if column[b] >= S else np.eye(S)[column[b]]) for r, (b, _, _) in enumerate(rows) if b < 4}
    outcomes, probs = anc.enumerate_joint([r[1] for r in rows], [None] + [mats[r[2]] for r in rows[1:]], tipL, w,
                                          model.getFrequencies())
    internal = [r for r in range(len(rows)) if r not in tipL]
    index = {o: k for k, o in enumerate(outcomes)}
    got = np.zeros(len(outcomes))
    for p in range(P):
        got[index[(int(cats[p]),) + tuple(int(states[r, p]) for r in internal)]] += 1.0 / P
    bound = 5 * np.sqrt(probs * (1 - probs) / P) + 3.0 / P
    assert np.all(np.abs(got - probs) <= bound), np.max(np.abs(got - probs) / bound)


def test_host_row_rules():
    build.build_engine()
    ok = beagle.checkAncestralRows
    nb, pr, mi = [6, 5, 3, 2, 4, 1, 0], [-1, 0, 1, 1, 0, 4, 4], [0, 5, 3, 2, 4, 1, 0]
    R = beagle.BeagleErrorCode.OUT_OF_RANGE_ERROR
    assert ok(nb, pr, mi, 7, 6) == 0
    assert ok([99] + nb[1:], pr, [-5] + mi[1:], 7, 6) == 0         # row 0's buffer and matrix are not read
    assert ok(nb, [0] + pr[1:], mi, 7, 6) == R                      # the root has no parent
    assert ok(nb, pr[:5] + [5, 4], mi, 7, 6) == R                   # a row as its own parent
    assert ok(nb, pr[:1] + [4] + pr[2:], mi, 7, 6) == R             # parent after the child
    assert ok(nb[:3] + [7] + nb[4:], pr, mi, 7, 6) == R             # buffer out of range
    assert ok(nb, pr, mi[:3] + [6] + mi[4:], 7, 6) == R             # matrix out of range
    assert ok([], [], [], 7, 6) == R
