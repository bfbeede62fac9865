"""Host logic of the 4-state walk route (no GPU, walk4e.cu::walk4Route through b200DebugWalkRoute): which kernel family runs
a phase, with how many patterns per thread (R), and whether the phase is thin.  The planner and both launchers take the
route from that one function; this restates the rule independently and sweeps it."""
import itertools

import numpy as np
import pytest

from beast_mcmc_b200 import beagle, build

MATRIX, EIGEN_PREDICATED, EIGEN_ALIGNED, STAGED, STAGED_VIRTUAL, UNSERVABLE = range(6)


@pytest.fixture(scope="module")
def lib():
    build.build_engine()
    return beagle.load_library()


def engine_route(lib, cp, ppad, sms, walk_r, thin_r1, single, n_subs, window, eigen, aligned, virt):
    out = np.zeros(3, dtype=np.int32)
    rc = lib.b200DebugWalkRoute(cp, ppad, sms, walk_r, thin_r1, single, n_subs, window, eigen, aligned, virt,
                                out.ctypes.data_as(beagle._IP))
    assert rc == 0
    return int(out[0]), int(out[1]), bool(out[2])


def expected_route(cp, ppad, sms, walk_r, thin_r1, single, n_subs, window, eigen, aligned, virt):
    g = 32 // cp
    thin = n_subs * -(-window // (g * walk_r)) < sms * 8          # few walks in flight
    if not eigen:
        r = 1 if thin_r1 and thin else walk_r
        # fp32 storage exists for CP <= 8 only; only the staged eigen-form kernels read virtual cherries
        return (UNSERVABLE if virt or (single and cp > 8) else MATRIX), r, thin
    if (thin_r1 and thin) or walk_r == 1:
        r = 1
    elif cp == 4 and walk_r == 2:
        r = 2
    else:
        r = 4
    if single and cp > 8:
        return UNSERVABLE, r, thin
    whole = aligned and ppad % (g * r) == 0
    if whole and cp <= 8 and g * r >= 4:
        return (STAGED_VIRTUAL if virt else STAGED), r, thin
    if virt:
        return UNSERVABLE, r, thin
    return (EIGEN_ALIGNED if whole and cp > 8 else EIGEN_PREDICATED), r, thin


# Ppad: multiples of 32 that are not multiples of 64, of 64 but not 128, and of 128
PPADS = [32, 96, 1056, 64, 320, 1088, 128, 1280, 50048]
# (subtree walks, SMs): empty, thin and wide phases on a full and a small device
SHAPES = [(0, 132), (1, 132), (7, 132), (64, 132), (500, 132), (3, 16), (40, 16)]


def sweep():
    """(args of b200DebugWalkRoute, expected route) over every category padding, walkR, rule switch, precision, list
    kind and phase shape"""
    for cp, walk_r, thin_r1, single, aligned, virt, eigen in itertools.product(
            [1, 2, 4, 8, 16, 32], [1, 2, 4], [0, 1], [0, 1], [0, 1], [0, 1], [0, 1]):
        for ppad in PPADS:
            # aligned lists span the padded axis; pattern-window lists are planned over their widest partition
            for window in ([ppad] if aligned else [ppad, max(1, ppad // 3 + 5)]):
                for n_subs, sms in SHAPES:
                    args = (cp, ppad, sms, walk_r, thin_r1, single, n_subs, window, eigen, aligned, virt)
                    yield args, expected_route(*args)


def test_route_table(lib):
    seen = set()
    for args, want in sweep():
        assert engine_route(lib, *args) == want, args
        seen.add((want[0], want[1]))
    # every family is reached, at every R it is built for
    assert {k for k, _ in seen} == set(range(6))
    assert {r for k, r in seen if k == STAGED_VIRTUAL} == {1, 2, 4}


def test_route_rejects_what_no_instance_has(lib):
    out = np.zeros(3, dtype=np.int32).ctypes.data_as(beagle._IP)
    assert lib.b200DebugWalkRoute(4, 128, 132, 4, 1, 0, 1, 128, 1, 1, 0, out) == 0
    for bad in [dict(cp=3), dict(cp=0), dict(cp=64), dict(walk_r=8), dict(ppad=0), dict(sms=0), dict(n_subs=-1),
                dict(window=0)]:
        a = dict(cp=4, ppad=128, sms=132, walk_r=4, n_subs=1, window=128) | bad
        rc = lib.b200DebugWalkRoute(a["cp"], a["ppad"], a["sms"], a["walk_r"], 1, 0, a["n_subs"], a["window"], 1, 1, 0, out)
        assert rc == beagle.BeagleErrorCode.OUT_OF_RANGE_ERROR, bad


def test_gpu_walk_cases_cover_every_cell(lib):
    """tests/test_gpu_walk_routes.py checks the walk against the oracle one (family, CP, R, precision) cell per row of its
    CASES.  Every row must reach the cell it names, and the rows together must reach every cell a phase can be routed
    to, each at least once with a pattern window that makes every lane and r slot of a warp live (G * R patterns, G =
    32 / CP) and leaves a partly live warp.  So a kernel instance added to walk4Route fails here until a case runs it, and
    so does a cell whose only wide row is deleted.  Rows beyond those (one live pattern, full category lanes, S < 4,
    aligned lists on the predicated kernel, the two rows on default rules) are extras; the guard asserts each kind is
    present, not each row."""
    from test_gpu_walk_routes import CASES, MATRIX, STAGED_VIRTUAL, _live, _parts, _ppad
    sms = 132                                             # H100 SXM; no row's route depends on it (see below)
    covered, wide = set(), set()
    for c in CASES:
        ppad = _ppad(c.P)
        window = ppad if c.lists == "aligned" else max(_parts(c.P))
        virt = int(c.family == STAGED_VIRTUAL)
        if c.natural:
            # the default rules: c.r is the walkR the instance picks (the GPU test reads it back from the plan line); a
            # wide phase
            assert c.env == {}, c
            args = (c.cp, ppad, sms, c.r, 1, int(c.single), 4096, window, 1, 1, virt)
        else:
            assert c.env["B200_WALK_R"] == str(c.r) and c.env["B200_THIN_R1"] == "0", c
            eigen = int(c.family != MATRIX and c.env.get("B200_EIGEN_WALK") != "0" and c.matrices == "eigen")
            assert eigen == int(c.family != MATRIX), c
            args = (c.cp, ppad, sms, c.r, 0, int(c.single), 1, window, eigen, int(c.lists == "aligned"), virt)
        assert c.cp == (1 << (c.C - 1).bit_length()) and c.S <= 4, c
        kernel, r, _ = engine_route(lib, *args)
        assert (kernel, r) == (c.family, c.r), (c, kernel, r)
        cell = (c.family, c.cp, c.r, c.single)
        covered.add(cell)
        g_r, live = 32 // c.cp * c.r, _live(c.P, c.lists)
        if live >= g_r and (live % g_r != 0 or g_r == 1):
            wide.add(cell)
    servable = {(want[0], args[0], want[1], bool(args[5])) for args, want in sweep() if want[0] != UNSERVABLE}
    assert servable <= covered, sorted(servable - covered)
    assert wide == covered, sorted(covered - wide)
    # the kinds of extra rows
    assert {(c.family, c.cp) for c in CASES if c.scale} == {(f, cp) for f, cp, _, _ in covered}
    assert {c.scale for c in CASES} == {None, "write", "cum"} and {c.log for c in CASES if c.scale} == {False, True}
    assert {c.C for c in CASES if c.C == c.cp} >= {4, 8} and {c.S for c in CASES} == {2, 3, 4}
    assert {c.P for c in CASES} >= {1, 33, 96, 301, 1000}
    assert {c.family for c in CASES if c.P == 1} == {MATRIX, EIGEN_PREDICATED, EIGEN_ALIGNED, STAGED, STAGED_VIRTUAL}
    assert {(c.cp, c.r) for c in CASES if c.family == EIGEN_PREDICATED and c.lists == "aligned"} == {(1, 4), (2, 4)}
    assert len([c for c in CASES if c.natural]) == 2
