"""The k-epsilon wall functions and fvMatrix::setValues on the CPU: oracle/wallfn_oracle.py against the reference's own setValues
(oracle/_ref/libref_setvalues.so), the host build of csrc/wallfn_kernels.cuh and of the setValues kernels of
csrc/fvmatrix_kernels.cuh against the oracle, yPlusLam and nutk, the corner weights, the near-wall distance, and three
wall-function kEpsilon::correct() calls on the oracle-backed stand-in in lockstep with the oracle."""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np
import pytest

import polymesh_cases as pc
import test_gpu_kepsilon_wall_functions as gw
import wallfn_backend
from oracle import fvm_oracle as fo
from oracle import ref_ldu as rl
from oracle import wallfn_oracle as wo
from test_foamfile_cpu import _scrambled
from test_gpu_engine_streams import Mismatches
from test_host_kernels_cpu import Host, _d

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_kernels", "wallfn_harness.cpp")
OUT = os.path.join(HERE, "host_kernels", "_build", "libhostk_wallfn.so")
CSRC = os.path.join(os.path.dirname(HERE), "rapidcfd-dev_b200", "csrc")
needs_ref = pytest.mark.skipif(not (rl.available() and os.path.exists(wo._LIB_SV)), reason="oracle/_ref/libref_setvalues.so not built")


@pytest.fixture(scope="module")
def hw():
    deps = [SRC, os.path.join(HERE, "host_kernels", "harness.cpp")] + [os.path.join(CSRC, f) for f in ("fvmatrix_kernels.cuh",
                                                                                                     "wallfn_kernels.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
                               "-Wno-unknown-pragmas", "-I", CSRC, "-shared", "-o", OUT, SRC])
    return C.CDLL(OUT)


def _meshes(meshmod):
    m = meshmod.hex_mesh(5)
    b = pc.refined_box(4, "random", seed=3)
    return [("hex", m.nCells, m.lower, m.upper, [p.faceCells for p in m.patches]),
            ("split-hex", b.nCells, b.lower, b.upper, [p.faceCells for p in b.wall_patches()])]


def _matrix(n, nF, nB, sym, seed):
    rng = np.random.default_rng(seed)
    return dict(diag=rng.uniform(5, 6, n), upper=rng.uniform(-1, 0, nF), lower=None if sym else rng.uniform(-1, 0, nF),
                source=rng.uniform(-1, 1, n), psi=rng.uniform(0, 1, n), ic=rng.uniform(0, 1, nB), bc=rng.uniform(0, 1, nB))


# ---- setValues ---------------------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("sym", [True, False], ids=["symmetric", "asymmetric"])
def test_set_values_oracle_equals_the_reference(meshmod, orc, sym):
    """bit for bit: set cells as owners and as neighbours, cells on two patches (edges) and three (corners), two successive calls
    (the second sees what the first cleared), a cell listed twice, the boundary coefficients of set cells cleared"""
    for name, n, lower, upper, pf in _meshes(meshmod):
        bfc = np.concatenate(pf)
        d = _matrix(n, len(lower), len(bfc), sym, 7)
        calls = [(pf[0], np.full(len(pf[0]), 2.5)), (np.concatenate([pf[2], pf[2][:3]]), np.full(len(pf[2]) + 3, -1.25))]
        r = wo.ref_set_values(n, lower, upper, pf, d["psi"], d["diag"], d["upper"], d["lower"], d["source"], d["ic"], d["bc"], calls)
        om = fo.FvMatrix(orc, orc.Addr(n, lower, upper), 1, d["diag"], d["upper"], d["lower"], d["source"], d["psi"], np.ones(n), bfc,
                         d["ic"], d["bc"])
        for c, v in calls:
            wo.set_values(om, c, v)
        M = Mismatches()
        for k, got in (("psi", om.psi[:, 0]), ("diag", om.diag), ("upper", om.upper), ("lower", om.lower), ("source", om.source[:, 0]),
                       ("ic", om.ic[:, 0]), ("bc", om.bc[:, 0])):
            M.bits(got, r[k], f"{name}: {k}")
        M.check()
        assert r["asymmetric"], "the reference's setValues leaves every matrix asymmetric"
        mask = np.zeros(n, bool)
        mask[np.concatenate([c for c, _ in calls])] = True
        assert (om.ic[mask[bfc]] == 0).all() and (om.ic[~mask[bfc]] != 0).all()
        assert (om.upper[mask[np.asarray(lower)]] == 0).all() and (om.lower[mask[np.asarray(upper)]] == 0).all()


@pytest.mark.parametrize("sym", [True, False], ids=["symmetric", "asymmetric"])
def test_set_values_host_build_equals_the_oracle(hw, meshmod, orc, sym):
    for name, n, lower, upper, pf in _meshes(meshmod):
        bfc = np.concatenate(pf)
        d = _matrix(n, len(lower), len(bfc), sym, 8)
        a = orc.Addr(n, lower, upper)
        om = fo.FvMatrix(orc, a, 1, d["diag"], d["upper"], d["lower"], d["source"], d["psi"], np.ones(n), bfc, d["ic"], d["bc"])
        H = Host(a, dict(bfc=bfc, diag=d["diag"], upper=d["upper"], lower=d["lower"]))
        got = {k: np.array(d[k] if d[k] is not None else d["upper"], float) for k in ("psi", "upper", "lower", "source", "ic", "bc")}
        for p, v in ((0, 2.5), (2, -1.25)):
            cells, vals = np.ascontiguousarray(pf[p], np.int32), np.full(len(pf[p]), v)
            wo.set_values(om, cells, vals)
            hw.hk_set_values(H.p(), len(cells), _d(cells), _d(vals), _d(got["psi"]), _d(d["diag"]), _d(got["upper"]), _d(got["lower"]),
                             _d(got["source"]), _d(got["ic"]), _d(got["bc"]))
        M = Mismatches()
        for k, ref in (("psi", om.psi[:, 0]), ("upper", om.upper), ("lower", om.lower), ("source", om.source[:, 0]), ("ic", om.ic[:, 0]),
                       ("bc", om.bc[:, 0])):
            M.bits(got[k], ref, f"{name}: {k}")
        M.check()


# ---- wall functions ----------------------------------------------------------------------------------------------------------------
def test_y_plus_lam_and_nutk_on_both_sides():
    ypl = wo.y_plus_lam()
    assert ypl == pytest.approx(11.53, abs=0.01)
    assert abs(ypl - np.log(9.8 * ypl) / 0.41) < 1e-3      # ten steps come close to the fixed point yPlus = log(E*yPlus)/kappa
    Cmu25, _ = wo.constants()
    nu, y = 1e-3, 0.01
    kLam = (ypl * nu / (Cmu25 * y)) ** 2                  # yPlus == yPlusLam
    k = np.array([0.5 * kLam, kLam * (1 - 1e-9), kLam * (1 + 1e-6), 4 * kLam])
    nut = wo.nutk(np.full(4, y), k, nu, ypl, Cmu25)
    assert (nut[:2] == 0).all() and (nut[2:] > 0).all()
    yPlus = Cmu25 * y * np.sqrt(k[3]) / nu
    assert nut[3] == pytest.approx(nu * (yPlus * 0.41 / np.log(9.8 * yPlus) - 1), rel=1e-14)


def test_corner_weights_in_the_cavity(meshmod):
    m, ps, types, y = gw.cavity_walls(meshmod, 4)
    bfc = np.concatenate([p.faceCells for p in m.patches]).astype(np.int64)
    allWalls = np.ones(len(bfc), bool)
    w = wo.corner_weights(m.nCells, bfc, allWalls)
    ijk = lambda i, j, k: i + 4 * (j + 4 * k)
    at = lambda c: set(w[bfc == c])
    assert at(ijk(1, 1, 0)) == {1.0} and at(ijk(1, 0, 0)) == {0.5} and at(ijk(0, 0, 0)) == {1.0 / 3.0}
    eps = np.repeat([t == "epsilonWallFunction" for t in types["epsTypes"]], np.diff(ps))
    w5 = wo.corner_weights(m.nCells, bfc, eps)            # the last patch is no epsilon wall: its faces carry 0, its cells count less
    assert (w5[~eps] == 0).all() and (w5[eps] > 0).all()
    kem = importlib.import_module("rapidcfd-dev_b200.kepsilon")
    assert np.array_equal(kem.corner_weights(m.nCells, bfc, eps), w5)


def test_wall_kernels_host_build_equal_the_oracle(hw, meshmod, orc):
    c = gw._entry_case(meshmod, orc)
    ref = gw._oracle_entries(orc, c)
    a = orc.Addr(c["n"], c["m"].lower, c["m"].upper)
    H = Host(a, dict(bfc=c["bfc"], diag=c["diag"], upper=c["upper"], lower=c["lower"]))
    Cmu25, Cmu75 = wo.constants()
    nutB = c["nutB"].copy()
    f = np.ascontiguousarray(c["nutkFaces"], np.int32)
    bfc = np.ascontiguousarray(c["bfc"], np.int32)
    hw.hk_nutk(len(f), _d(f), _d(bfc), _d(c["y"]), _d(c["k"]), C.c_double(0.01), C.c_double(wo.y_plus_lam()), C.c_double(Cmu25),
               C.c_double(wo.KAPPA), C.c_double(wo.E), _d(nutB))
    G, eps, epsB = c["G"].copy(), c["eps"].copy(), c["epsB"].copy()
    hw.hk_epsilon_wall(H.p(), _d(c["cw"]), _d(c["y"]), _d(c["k"]), _d(c["U"]), _d(c["Ub"]), _d(c["bDelta"]), _d(c["nutB"]),
                       C.c_double(0.01), C.c_double(Cmu25), C.c_double(Cmu75), C.c_double(wo.KAPPA), _d(G), _d(eps), _d(epsB))
    M = Mismatches()
    for k, got in (("nutB", nutB), ("G", G), ("eps", eps), ("epsB", epsB)):
        M.bits(got, ref[k], k)
    M.check()
    assert (nutB[f] == 0).any() and (nutB[f] > 0).any()


# ---- near-wall distance ------------------------------------------------------------------------------------------------------------
def test_near_wall_dist_on_a_box(meshmod):
    ff = importlib.import_module("rapidcfd-dev_b200.foamfile")
    m = meshmod.hex_mesh(4, 3, 5)
    y = ff.from_hex_mesh(m).near_wall_dist([p.name for p in m.patches])
    np.testing.assert_allclose(y, m.h / 2, rtol=1e-14)


def test_near_wall_dist_on_a_skewed_mesh_matches_brute_force(meshmod):
    ff = importlib.import_module("rapidcfd-dev_b200.foamfile")
    pm, hm = _scrambled(ff, meshmod, (5, 4, 3), 3, skew=0.6)
    y = pm.near_wall_dist([p.name for p in pm.patches])
    C, _ = pm.cell_centres_and_volumes()
    nI = pm.nInternalFaces
    for p in pm.patches:
        pts = [pm.points[pm.faceLabels[pm.faceOffsets[f]:pm.faceOffsets[f + 1]]] for f in range(p.startFace, p.startFace + p.nFaces)]
        for i in range(p.nFaces):
            brute = min(ff._face_distance(C[pm.owner[p.startFace + i]], q) for q in pts)
            assert y[p.startFace - nI + i] == brute
    assert not np.allclose(y, hm.h / 2)                     # the skew moved the centres off the half-spacing


# ---- the step ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [None, 0.7])
def test_kepsilon_wall_functions_stand_in_reproduces_the_oracle(monkeypatch, meshmod, orc, alpha):
    product, oracle, (bfc, ps) = gw.kepsilon_wall_case(meshmod, orc, 8, "upwind", alpha)
    L = gw.run_wall_lockstep(monkeypatch, wallfn_backend.fixture(), product, oracle)
    assert len(L.dev) == 6
    gw.check_wall_cells(L, bfc[:ps[-2]])


def test_patch_types_are_checked_by_name(meshmod, orc):
    capi, ctx, torch = wallfn_backend.fixture()
    ico = importlib.import_module("rapidcfd-dev_b200.icofoam")
    kem = importlib.import_module("rapidcfd-dev_b200.kepsilon")
    m, case = ico.cavity(capi, ctx, torch, 4)
    m, ps, types, y = gw.cavity_walls(meshmod, 4)
    nB, n = int(ps[-1]), m.nCells
    args = (np.full(nB, m.h * m.h), np.full(nB, 2.0 / m.h), np.full(n, 0.01), np.full(n, 0.1), np.full(nB, 0.01), np.full(nB, 0.1))
    bad = dict(types, epsTypes=["omegaWallFunction"] + types["epsTypes"][1:])
    with pytest.raises(ValueError, match="Unknown patchField type omegaWallFunction"):
        kem.KEpsilon(capi, case, *args, patchStart=ps, y=y, **bad)
