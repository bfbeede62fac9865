"""The JNI tier (libhmsbeagle-jni.so): exported symbol set and argument lists against the jar's
native descriptors (tests/golden/beagle_jar_abi.json), and a JVM-less drive of the exported
Java_beagle_BeagleJNIWrapper_* entry points through a fake JNIEnv."""
import json
import os
import re
import subprocess

import pytest

import helpers as H
from beast_mcmc_b200 import build

ROOT = H.ROOT
ABI = json.load(open(os.path.join(ROOT, "tests", "golden", "beagle_jar_abi.json")))
TYPE2DESC = {"jint": "I", "jlong": "J", "jdouble": "D", "jintArray": "[I", "jdoubleArray": "[D", "jobject": "L"}


@pytest.fixture(scope="module")
def jni(tmp_path_factory):
    build.build_engine()
    lib = build.build_jni()
    src = os.path.join(ROOT, "tests", "jni_fake", "fake_jvm.cpp")
    # built into this session's own temporary directory: the checkout may be read-only or shared with another run
    exe = str(tmp_path_factory.mktemp("jni_fake") / "fake_jvm")
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", exe, src, "-ldl"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return lib, exe


def test_all_47_natives_exported(jni):
    lib, _ = jni
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    want = {"Java_beagle_BeagleJNIWrapper_" + n["name"] for n in ABI["natives"]}
    assert len(want) == 47
    assert want <= exported, sorted(want - exported)


def test_native_argument_lists_match_descriptors():
    src = open(os.path.join(ROOT, "beast-mcmc_b200", "csrc", "jni_shim.cpp")).read()
    defs = dict()
    for m in re.finditer(r"NATIVE\((\w+), (\w+)\)\(([^)]*)\)", src):
        ret, name, args = m.group(1), m.group(2), m.group(3)
        types = [a.strip().split()[0] for a in args.split(",")]
        assert types[0] == "JNIEnv*" and types[1] == "jobject", name     # instance method of the singleton
        defs[name] = (ret, types[2:])
    for n in ABI["natives"]:
        ret, types = defs[n["name"]]
        params, rdesc = re.match(r"\((.*)\)(.*)", n["descriptor"]).groups()
        params = re.sub(r"L[^;]+;", "L", params)
        got = "".join(TYPE2DESC[t] for t in types)
        assert got == params, (n["name"], got, params)
        assert {"I": "jint"}.get(rdesc, "jstring" if "String" in rdesc else "jobjectArray") == ret, n["name"]


def test_fake_jvm_info(jni):
    lib, exe = jni
    out = subprocess.run([exe, lib, "info"], capture_output=True, text=True, check=True).stdout
    assert re.search(r"version (\d+)\.\d+\.\d+", out) and int(re.search(r"version (\d+)", out).group(1)) >= 4
    assert "resource 0 name=CPU" in out


@pytest.mark.gpu
def test_fake_jvm_tiny_test(jni, tmp_path):
    """BeagleFactory.main's tiny test through the JNI entry points: PAUP logL -1574.63623."""
    lib, exe = jni
    tree, pats, model, site, expected = H.tiny_case()
    fx = tmp_path / "tiny.txt"
    with open(fx, "w") as f:
        f.write(f"3 {pats.patternCount}\n")
        for t in range(3):
            f.write(" ".join(str(int(s)) for s in pats.states[t]) + "\n")
    out = subprocess.run([exe, lib, "tiny", str(fx)], capture_output=True, text=True, check=True).stdout
    assert f"logL {expected:.5f} rc 0" in out, out
    assert "impl=B200-CUDA-Double" in out


@pytest.mark.gpu
def test_fake_jvm_gradient_natives(jni, tmp_path):
    """updatePrePartials / setDifferentialMatrix / calculateEdgeDifferentials / calculateCrossProductDifferentials through
    the JNI entry points (null output array, in/out array) against the oracle driven with the same calls."""
    import numpy as np
    from oracle.felsenstein import OracleBeagle
    lib, exe = jni
    tree, pats, model, site, expected = H.tiny_case()
    fx = tmp_path / "tiny.txt"
    with open(fx, "w") as f:
        f.write(f"3 {pats.patternCount}\n")
        for t in range(3):
            f.write(" ".join(str(int(s)) for s in pats.states[t]) + "\n")
    out = subprocess.run([exe, lib, "gradient", str(fx)], capture_output=True, text=True, check=True).stdout
    P = pats.patternCount
    o = OracleBeagle(3, 7, 3, 4, P, 1, 5, 1, 0)
    for t in range(3):
        o.setTipStates(t, pats.states[t])
    o.setPatternWeights(np.ones(P))
    e = model.getEigenDecomposition()
    o.setEigenDecomposition(0, e.Evec, e.Ievc, e.Eval)
    o.setCategoryRates(np.ones(1)); o.setCategoryWeights(0, np.ones(1)); o.setStateFrequencies(0, np.full(4, 0.25))
    I = lambda *v: np.asarray(v, dtype=np.int32)
    lengths = np.array([0.1, 0.1, 0.2, 0.1])
    o.updateTransitionMatrices(0, I(0, 1, 2, 3), None, None, lengths, 4)
    o.updatePartials(I(3, -1, -1, 0, 0, 1, 1, 4, -1, -1, 2, 2, 3, 3), 2, -1)
    o.setPartials(9, np.full(4 * P, 0.25))
    o.updatePrePartials(I(8, -1, -1, 9, 3, 2, 2, 7, -1, -1, 9, 2, 3, 3, 5, -1, -1, 8, 0, 1, 1, 6, -1, -1, 8, 1, 0, 0), 4, -1)
    Q = np.full((4, 4), 1.0 / 3.0); np.fill_diagonal(Q, -1.0)
    o.setDifferentialMatrix(4, Q.reshape(-1))
    s1, s2 = np.zeros(4), np.zeros(4)
    o.calculateEdgeDifferentials(I(0, 1, 2, 3), I(5, 6, 7, 8), I(4, 4, 4, 4), I(0), 4, None, s1, s2)
    cross = np.zeros(16)
    o.calculateCrossProductDifferentials(I(0, 1, 2, 3), I(5, 6, 7, 8), I(0), I(0), lengths, 4, cross, None)
    edge = re.search(r"edge rc 0 (.*)", out).group(1).split()
    got_cross = re.search(r"cross rc 0 (.*)", out).group(1).split()
    assert np.allclose([float(v) for v in edge], s1, rtol=1e-8, atol=1e-8), (edge, s1)
    assert np.allclose([float(v) for v in got_cross], cross, rtol=1e-7, atol=2e-8), (got_cross, cross)
    assert f"logL {expected:.5f} rc 0" in out


@pytest.mark.gpu
def test_fake_jvm_beagle_auto(jni):
    """-beagle_auto (BDLD:400-434): getBenchmarkedResourceList returns the GPU resources, fastest first, never resource 0."""
    lib, exe = jni
    out = subprocess.run([exe, lib, "auto"], capture_output=True, text=True, check=True).stdout
    rows = re.findall(r"benchmarked (\d+) resource=(\d+) name=(.*) impl=B200-CUDA-Double rc=0 ms=([0-9.]+) ratio=([0-9.]+)", out)
    assert rows, out
    assert [int(r[0]) for r in rows] == list(range(len(rows)))
    assert all(int(r[1]) >= 1 for r in rows) and float(rows[0][4]) == 1.0
    ms = [float(r[3]) for r in rows]
    assert ms == sorted(ms) and ms[0] > 0.0
