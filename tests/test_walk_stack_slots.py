"""Host logic of the sibling stack (no GPU, api.cu::assignStackSlots through b200DebugStackSlots): inside one subtree walk
every slot a child is read from holds that child's value -- written earlier in the same walk and not reused in between --;
children taken from registers, tips and children from another walk never take a slot; at most three slots are used."""
import numpy as np
import pytest

from beast_mcmc_b200 import beagle, build
from test_plan_host_logic import tree_ops

DEPTH = 3
NOSLOT = 0xFF


@pytest.fixture(scope="module")
def lib():
    build.build_engine()
    return beagle.load_library()


def stack_plan(lib, ops, nbuf, tips, want=64, minT=4, small=24):
    ops = np.ascontiguousarray(ops, dtype=np.int32).reshape(-1)
    n = len(ops) // 7
    rec = np.zeros(5 * n, dtype=np.int32)
    subs = np.zeros(2 * n, dtype=np.int32)
    ph = np.zeros(n + 2, dtype=np.int32)
    cnt = np.zeros(5, dtype=np.int32)
    ip = lambda a: a.ctypes.data_as(beagle._IP)
    assert lib.b200DebugStackSlots(ip(ops), n, nbuf, tips, want, minT, small, ip(rec), ip(subs), ip(ph), ip(cnt)) == 0
    return rec.reshape(-1, 5), subs[:2 * cnt[0]].reshape(-1, 2), ph[:cnt[1] + 1], cnt


def check_slots(rec, subs):
    """replays every walk: returns (children read from a slot, internal children read from memory, deepest slot + 1)"""
    stack_reads = memory_reads = depth = 0
    for b, e in subs:
        slot_value = {}                   # slot -> buffer whose current value it holds
        produced = set()                  # buffers written earlier in this walk
        for pos in range(b, e):
            dest, c1, c2, flags, slots = (int(v) for v in rec[pos])
            src = (slots & 0xFF, (slots >> 8) & 0xFF)
            dst = (slots >> 16) & 0xFF
            for ch, child in enumerate((c1, c2)):
                from_registers = ch == 0 and flags & 2
                if child < 0 or from_registers:
                    assert src[ch] == NOSLOT                                  # tips and forwarded children: no slot
                    if from_registers:
                        assert pos > b and int(rec[pos - 1][0]) == child
                    continue
                if src[ch] == NOSLOT:
                    memory_reads += 1
                    continue
                stack_reads += 1
                assert child in produced                                      # never a child from another walk
                assert slot_value.get(src[ch]) == child                       # written earlier, not reused since
            for s in [s for s, buf in slot_value.items() if buf == dest]:     # the old value of dest is gone
                del slot_value[s]
            if dst != NOSLOT:
                assert dst < DEPTH
                later = [p for p in range(pos + 1, e)
                         if (int(rec[p][2]) == dest or (int(rec[p][1]) == dest and not rec[p][3] & 2))]
                assert later                                                  # only results that are read back later
                slot_value[dst] = dest
                depth = max(depth, dst + 1)
            produced.add(dest)
    return stack_reads, memory_reads, depth


@pytest.mark.parametrize("tips,seed,traversal", [(50, 3, "POST_ORDER"), (400, 4, "POST_ORDER"),
                                                 (1000, 5, "REVERSE_LEVEL_ORDER"), (1000, 6, "POST_ORDER")])
@pytest.mark.parametrize("want", [1, 64])
def test_slots_hold_what_is_read(lib, tips, seed, traversal, want):
    _, ops = tree_ops(tips, seed, traversal)
    rec, subs, phases, cnt = stack_plan(lib, ops, 2 * tips, tips, want=want)
    stack_reads, memory_reads, depth = check_slots(rec, subs)
    assert (stack_reads, memory_reads, depth) == (cnt[2], cnt[3], cnt[4])
    assert stack_reads > 0 and depth <= DEPTH
    if want == 1:                        # one walk for the whole tree: a memory read is an overflowed sibling
        assert len(subs) == 1


def test_cross_phase_children_read_from_memory(lib):
    """with many small subtrees, the results that cross a phase boundary are read from memory"""
    _, ops = tree_ops(1000, 7, "POST_ORDER")
    rec, subs, phases, cnt = stack_plan(lib, ops, 2000, 1000, want=64)
    assert len(phases) > 2 and cnt[3] > 0
    check_slots(rec, subs)


def test_overflow_and_rewrite(lib):
    """a caller-order list (a buffer written twice) that needs more than three live siblings"""
    T = 32
    ops = []
    nxt = T

    def balanced(lo, hi):
        nonlocal nxt
        if hi - lo == 1:
            return lo
        a, b = balanced(lo, (lo + hi) // 2), balanced((lo + hi) // 2, hi)
        ops.append([nxt, -1, -1, a, a, b, b])
        nxt += 1
        return nxt - 1
    root = balanced(0, T)
    ops.append(list(ops[0]))             # rewrites the first internal node: hazard, one walk in the caller's order
    ops.append([nxt, -1, -1, ops[0][0], 0, root, 0])
    rec, subs, phases, cnt = stack_plan(lib, np.array(ops), nxt + 1, T)
    assert len(subs) == 1
    stack_reads, memory_reads, depth = check_slots(rec, subs)
    assert (stack_reads, memory_reads, depth) == (cnt[2], cnt[3], cnt[4])
    assert depth == DEPTH and stack_reads > 0 and memory_reads > 0
