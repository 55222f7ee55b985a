"""The interFoam phase-fraction step without a GPU: the device bodies of csrc/vof_kernels.cuh executed on the host against the oracle
(bit for bit), the fused limited flux against the four-step composition, analytic checks of oracle/interfoam_oracle.py, the step
of rapidcfd-dev_b200/interfoam.py over the oracle-backed stand-in, the dictionary look-ups and the golden vectors."""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np
import pytest

import interfoam_backend
import interfoam_cases as ic
from oracle import interfoam_oracle as io
from oracle import limiters_oracle as lo
from test_fv_kernels_cpu import _cases
from test_host_kernels_cpu import CSRC, HERE, Host, _d

SRC = os.path.join(HERE, "host_kernels", "vof_harness.cpp")
OUT = os.path.join(HERE, "host_kernels", "_build", "libhostk_vof.so")
SCHEMES = sorted(lo.SCHEMES)


@pytest.fixture(scope="module")
def hkv():
    deps = [SRC, os.path.join(HERE, "host_kernels", "harness.cpp")] + \
           [os.path.join(CSRC, f) for f in ("vof_kernels.cuh", "fieldops_kernels.cuh", "fvmatrix_kernels.cuh", "mules_kernels.cuh", "fv_kernels.cuh")]
    if not os.path.exists(OUT) or any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps):
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
                               "-Wno-unknown-pragmas", "-I", CSRC, "-I", os.path.dirname(SRC), "-shared", "-o", OUT, SRC])
    L = C.CDLL(OUT)
    L.hk_limited_flux.argtypes = [C.c_int, C.c_int, C.c_double] + [C.c_void_p] * 7 + [C.c_int, C.c_int, C.c_void_p]
    L.hk_interface_flux.argtypes = [C.c_void_p] * 6 + [C.c_double, C.c_void_p, C.c_void_p, C.c_double] + [C.c_void_p] * 3
    return L


def _fields(m, seed):
    """random fields with what the branches need: cells of equal vf (the clipped branch of NVDTVD::r, gradf = 0), cells without
    gradient (mag(gradAlphaf) = 0: nHatfv = 0/(0 + deltaN)), fluxes of both signs and exactly zero"""
    rng = np.random.default_rng(seed)
    n, nF = m.nCells, m.nFaces
    vf, g = rng.uniform(0, 1, n), rng.uniform(-1, 1, (n, 3))
    flat = rng.uniform(0, 1, n) < 0.4
    vf[flat], g[flat] = 0.25, 0.0
    flux = rng.uniform(-1, 1, nF)
    flux[::7] = 0.0
    return dict(vf=vf, g=g, C=rng.uniform(0, 1, (n, 3)), cd=rng.uniform(0.3, 0.7, nF), flux=flux, Sf=rng.uniform(-1, 1, (nF, 3)),
                magSf=rng.uniform(0.5, 2, nF), w=rng.uniform(0, 1, nF))


def test_limited_flux_body_on_the_host(hkv, meshmod, orc):
    for name, m, bfc in _cases(meshmod):
        d = _fields(m, 21)
        l, u = np.ascontiguousarray(m.lower, np.int32), np.ascontiguousarray(m.upper, np.int32)
        clipped = np.abs((d["vf"][u] - d["vf"][l])) == 0
        assert clipped.any() and not clipped.all()
        for scheme in SCHEMES:
            for k in ((1.0, 0.3) if scheme == "limitedLinear" else (1.0,)):
                for fs in (1, -1):
                    for os_ in (1, -1):
                        out = np.zeros(m.nFaces)
                        hkv.hk_limited_flux(m.nFaces, lo.SCHEMES[scheme], 2.0 / max(k, lo.SMALL), _d(l), _d(u), _d(d["flux"]), _d(d["vf"]),
                                            _d(d["g"]), _d(d["C"]), _d(d["cd"]), fs, os_, _d(out))
                        want = io.limited_flux(scheme, l, u, d["flux"], d["vf"], d["g"], d["C"], d["cd"], k, fs, os_)
                        assert np.array_equal(out, want), (name, scheme, k, fs, os_)


@pytest.mark.parametrize("scheme", SCHEMES)
def test_limited_flux_equals_the_four_step_composition(meshmod, orc, scheme):
    """limiter -> limited weights -> interpolate(vf, weights) -> faceFlux*face, each through the primitive that checks the entry
    point of that step, against the oracle of the fused pass"""
    for name, m, bfc in _cases(meshmod):
        d = _fields(m, 22)
        a = orc.Addr(m.nCells, m.lower, m.upper)
        for fs, os_ in ((1, 1), (-1, -1), (-1, 1)):
            F = fs * d["flux"]
            lim = lo.limiter(scheme, m.lower, m.upper, F, d["vf"], d["g"], d["C"], 0.5)
            face = np.asarray(orc.interpolate_linear(a, lo.limited_weights(F, lim, d["cd"]), d["vf"], 1))
            want = os_ * (F * face)
            got = io.limited_flux(scheme, m.lower, m.upper, d["flux"], d["vf"], d["g"], d["C"], d["cd"], 0.5, fs, os_)
            assert np.array_equal(got, want), (name, fs, os_)


def test_interface_flux_bodies_on_the_host(hkv, meshmod, orc):
    for name, m, bfc in _cases(meshmod):
        d = _fields(m, 23)
        rng = np.random.default_rng(24)
        nB = len(bfc)
        a = orc.Addr(m.nCells, m.lower, m.upper)
        H = Host(a, dict(bfc=bfc, diag=np.zeros(m.nCells), upper=np.zeros(m.nFaces), lower=None))
        bSf, bSn = rng.uniform(-1, 1, (max(nB, 1), 3)), rng.uniform(-1, 1, max(nB, 1))
        bSn[::3] = 0.0
        for deltaN in (1e-8 / 0.1, 0.5):
            for withPhi in (False, True):
                nHatf, nHatfB, phir = np.zeros(m.nFaces), np.zeros(max(nB, 1)), np.full(m.nFaces, -7.0)
                hkv.hk_interface_flux(H.p(), _d(d["w"]), _d(d["g"]), _d(d["Sf"]), _d(bSf), _d(bSn), deltaN, _d(d["flux"]) if withPhi else None,
                                      _d(d["magSf"]), 0.75, _d(nHatf), _d(nHatfB), _d(phir))
                w0, w1, w2 = io.interface_flux(m.lower, m.upper, d["w"], d["g"], d["Sf"], bfc, bSf[:nB], bSn[:nB], deltaN,
                                               d["flux"] if withPhi else None, d["magSf"], 0.75)
                assert np.array_equal(nHatf, w0) and np.array_equal(nHatfB[:nB], w1), (name, deltaN)
                assert np.array_equal(phir, w2) if withPhi else (phir == -7.0).all(), name
                flatFaces = ~d["g"][m.lower].any(1) & ~d["g"][m.upper].any(1)
                assert flatFaces.any() and not nHatf[flatFaces].any()          # 0/(0 + deltaN) = 0, no NaN
                assert np.isfinite(nHatf).all() and np.isfinite(nHatfB).all()


# ---- analytic checks of the oracle ------------------------------------------------------------------------------------------
def test_planar_interface_has_unit_normal_and_no_curvature(meshmod, orc):
    m = meshmod.hex_mesh(16)
    nrm = np.array([1.0, 2.0, 0.5]) / np.linalg.norm([1.0, 2.0, 0.5])
    dist = (m.cell_centres() - 0.5) @ nrm
    interior = np.ones(m.nCells, bool)
    interior[np.concatenate([p.faceCells for p in m.wall_patches()])] = False
    faces = interior[m.lower] & interior[m.upper] & (np.abs(0.5 * (dist[m.lower] + dist[m.upper])) < 2 * m.h)
    assert faces.sum() > 100
    tight = ic.oracle(orc, m, 0.5 + dist, 1.0)                     # a plane: constant gradient away from the walls
    assert np.abs(tight.nHatf[faces] - m.Sf()[faces] @ nrm).max() <= 1e-6 * m.h ** 2
    ijk = np.floor(m.cell_centres() / m.h).astype(int)              # the wall cells' zeroGradient gradient reaches one cell further
    cells = ((ijk >= 2) & (ijk <= 13)).all(1) & (np.abs(dist) < 2 * m.h)
    assert cells.sum() > 100
    assert np.abs(tight.K[cells]).max() <= 1e-6


def test_sphere_curvature_and_compression_flux(meshmod, orc):
    m = meshmod.hex_mesh(48)
    R = 0.25
    o = ic.oracle(orc, m, ic.sphere(m, (0.5, 0.5, 0.5), R, 1.5), 1.0)
    cells = (o.alpha1 > 0.1) & (o.alpha1 < 0.9)
    assert cells.sum() > 1000
    # K = -div(nHat), nHat = grad(alpha)/|grad(alpha)| pointing inward: 2/R
    assert abs(o.K[cells].mean() - 2.0 / R) <= 0.1 * 2.0 / R
    phi, _ = ic.rotation_flux(m)
    _, _, phir = io.interface_flux(m.lower, m.upper, o.w, o.gradAlpha, o.Sf, o.bfc, o.bSf, np.zeros(len(o.bfc)), o.deltaN, phi, o.magSf, 0.8)
    assert np.array_equal(np.sign(phir), np.sign(o.nHatf) * (phi != 0))
    assert np.allclose(np.abs(phir), 0.8 * np.abs(phi) * np.abs(o.nHatf) / o.magSf, rtol=1e-14, atol=0)
    assert np.array_equal(o.near_interface(), ((o.alpha1 >= 0.01) & (o.alpha1 <= 0.99)).astype(float))
    assert o.surface_tension_force().shape == (m.nFaces,)


# ---- the step -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("MULESCorr", [False, True])
@pytest.mark.parametrize("nAlphaCorr,nSub", [(1, 1), (2, 1), (1, 2), (2, 2)])
def test_step_is_bounded_and_conservative(meshmod, orc, MULESCorr, nAlphaCorr, nSub):
    m = meshmod.hex_mesh(24)
    a0, V = ic.sphere(m), m.volumes()
    o = ic.run_oracle(orc, m, a0, ic.controls(MULESCorr, nAlphaCorr, nSub), 3, ic.SOLVER)
    assert o.alpha1.min() >= -1e-10 and o.alpha1.max() <= 1 + 1e-10
    # closed box: the explicit updates conserve to rounding, the predictor of the MULESCorr branch to its solver tolerance
    assert abs((o.alpha1 * V).sum() - (a0 * V).sum()) <= (1e-9 if MULESCorr else 1e-12) * (a0 * V).sum()
    assert np.array_equal(o.rho, o.alpha1 * ic.RHO1 + o.alpha2 * ic.RHO2) and np.array_equal(o.alpha2, 1.0 - o.alpha1)
    assert len(o.reports) == 3 * nSub * (2 if MULESCorr else 1)
    assert abs(o.reports[-1][0] - (o.alpha1 * V).sum() / V.sum()) <= 1e-15


def test_rho_phi_of_two_sub_cycles_is_the_weighted_sum(meshmod, orc):
    m = meshmod.hex_mesh(24)
    a0 = ic.sphere(m)
    phi, dt = ic.rotation_flux(m)
    zB = np.zeros(6 * 24 * 24)
    whole = ic.oracle(orc, m, a0, 1.0)
    whole.alpha_eqn_sub_cycle(phi, zB, dt, ic.controls(nAlphaSubCycles=2), ic.RHO1, ic.RHO2)
    parts = ic.oracle(orc, m, a0, 1.0)
    s = 0.0 * phi
    for _ in range(2):
        parts.alpha_eqn(phi, zB, dt / 2, ic.controls(), ic.RHO1, ic.RHO2)
        s = s + ((dt / 2) / dt) * parts.rhoPhi
    assert np.array_equal(whole.rhoPhi, s) and np.array_equal(whole.alpha1, parts.alpha1)


def test_compression_narrows_the_interface(meshmod, orc):
    m = meshmod.hex_mesh(24)
    a0 = ic.sphere(m, width=1.5)
    n = {c: ic.band(ic.run_oracle(orc, m, a0, ic.controls(cAlpha=c), 20).alpha1) for c in (0.0, 1.0)}
    assert n[1.0] < n[0.0], n


# ---- the sequencing of rapidcfd-dev_b200/interfoam.py over the stand-in -------------------------------------------------------
@pytest.mark.parametrize("MULESCorr,prevCorr", [(False, False), (True, False), (True, True)])
def test_standin_dry_run_equals_the_oracle(meshmod, orc, MULESCorr, prevCorr):
    capi, ctx, torch = interfoam_backend.fixture()
    m = meshmod.hex_mesh(12)
    a0 = ic.sphere(m)
    ctl = ic.controls(MULESCorr, 2, 2, alphaApplyPrevCorr=prevCorr)
    mesh, mix, ph = ic.run_product(capi, ctx, torch, m, a0, ctl, 3, ic.SOLVER)
    o = ic.run_oracle(orc, m, a0, ctl, 3, ic.SOLVER)
    got = {k: getattr(ph, k).numpy() for k in ("alpha1", "alpha2", "rhoPhi", "rhoPhiB", "rho")}
    got.update(K=mix.K.numpy(), nHatf=mix.nHatf.numpy(), stf=mix.surface_tension_force().numpy(), near=mix.near_interface().numpy())
    want = dict(alpha1=o.alpha1, alpha2=o.alpha2, rhoPhi=o.rhoPhi, rhoPhiB=o.rhoPhiB, rho=o.rho, K=o.K, nHatf=o.nHatf,
                stf=o.surface_tension_force(), near=o.near_interface())
    for k in want:
        if MULESCorr:      # one linear solve per pass
            assert np.allclose(got[k], want[k], rtol=0, atol=1e-10 * max(1.0, np.abs(want[k]).max())), k
        else:
            assert np.array_equal(got[k], want[k]), k
    assert np.allclose(ph.reports, o.reports, rtol=0, atol=1e-10) and mesh.deltaN == o.deltaN


# ---- dictionaries -------------------------------------------------------------------------------------------------------------
FVSOLUTION = """solvers { "alpha.water.*" { nAlphaCorr 2; nAlphaSubCycles 3; cAlpha 1; %s
    solver smoothSolver; smoother GaussSeidel; tolerance 1e-8; relTol 0; } }"""
FVSCHEMES = "ddtSchemes { default Euler; } divSchemes { default none; div(phi,alpha) Gauss %s; div(phirb,alpha) Gauss %s; }"


def test_dictionary_lookups_and_refusals():
    ff = importlib.import_module("rapidcfd-dev_b200.foamfile")
    itf = importlib.import_module("rapidcfd-dev_b200.interfoam")
    sch = ff.FvSchemes(ff.parse_dict(FVSCHEMES % ("vanLeer", "limitedLinear 0.5")))
    c = ff.alpha_controls(ff.parse_dict(FVSOLUTION % ""), sch)
    assert c == dict(nAlphaCorr=2, nAlphaSubCycles=3, cAlpha=1.0, MULESCorr=False, alphaApplyPrevCorr=False, icAlpha=0.0, nLimiterIter=3,
                     extremaCoeff=0.0, alphaScheme=("vanLeer", 1.0), alpharScheme=("limitedLinear", 0.5))
    itf.refuse_unsupported(c, ["zeroGradient"], sch.ddt("ddt(alpha)")[0])
    c = ff.alpha_controls(ff.parse_dict(FVSOLUTION % "MULESCorr yes; nLimiterIter 5; extremaCoeff 0.1; alphaApplyPrevCorr on;"), sch)
    assert (c["MULESCorr"], c["nLimiterIter"], c["extremaCoeff"], c["alphaApplyPrevCorr"]) == (True, 5, 0.1, True)
    assert ff.solver_controls(ff.parse_dict(FVSOLUTION % ""), "alpha.water")[:2] == ("smoothSolver", "GaussSeidel")
    with pytest.raises(KeyError, match="nLimiterIter"):                     # CMULES looks it up without a default
        ff.alpha_controls(ff.parse_dict(FVSOLUTION % "MULESCorr yes;"), sch)
    with pytest.raises(KeyError, match="cAlpha"):
        ff.alpha_controls(ff.parse_dict(FVSOLUTION.replace("cAlpha 1;", "") % ""), sch)
    with pytest.raises(ValueError, match="Unknown discretisation scheme SuperBee"):
        ff.alpha_controls(ff.parse_dict(FVSOLUTION % ""), ff.FvSchemes(ff.parse_dict(FVSCHEMES % ("SuperBee", "linear"))))
    with pytest.raises(KeyError, match=r"div\(phirb,alpha\)"):
        ff.alpha_controls(ff.parse_dict(FVSOLUTION % ""), ff.FvSchemes(ff.parse_dict("divSchemes { default none; div(phi,alpha) Gauss upwind; }")))
    ok = ic.controls()
    for kw, word in ((dict(controls=dict(ok, icAlpha=0.2)), "icAlpha"), (dict(ddtScheme="localEuler"), "LTSSOLVE"),
                     (dict(alphaPatchTypes=["zeroGradient", "constantAlphaContactAngle"]), "correctContactAngle"),
                     (dict(alphaPatchTypes=["inletOutlet"]), "inletOutlet"), (dict(movingMesh=True), "moving mesh"),
                     (dict(nCoupledFaces=4), "coupled")):
        with pytest.raises(NotImplementedError, match=word):
            itf.refuse_unsupported(**dict(dict(controls=ok), **kw))
    with pytest.raises(ValueError, match="Unknown discretisation scheme QUICK"):
        itf.refuse_unsupported(dict(ok, alpharScheme=("QUICK", 1.0)))


# ---- golden vectors ---------------------------------------------------------------------------------------------------------
def test_oracle_matches_its_golden_vectors(orc):
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    try:
        mg = importlib.import_module("make_interfoam_golden")
    finally:
        sys.path.pop(0)
    want = np.load(os.path.join(HERE, "golden", "interfoam_golden.npz"))
    got = mg.compute()
    assert sorted(got) == sorted(want.files)
    for k in ("nHatf", "nHatfB", "K", "phir", "alpha_explicit"):
        assert np.array_equal(got[k], want[k]), k
    assert np.allclose(got["alpha_mulescorr"], want["alpha_mulescorr"], rtol=0, atol=1e-10)
