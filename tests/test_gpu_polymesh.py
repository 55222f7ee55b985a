"""The cell-walking kernels, the asymmetric engine and GAMG on the device on split-hex polyhedral meshes (tests/polymesh_cases.py):
cells with up to 24 owner or losort faces, six boundary faces in four patches and four coupled faces, and a random graph with cells
without faces.  A hex box never has more than three faces per side, so the loops after the prefetched first batch of the face-sum
(fv_kernels.cuh), H / relax (fvmatrix_kernels.cuh) and MULES kernels, and the per-cell lists the library builds
(b200ldu_fv_boundary_set, the coupled-face lists of the layout builder), run here for the first time on the GPU.

Everything that is a sum of separately rounded terms in the reference's order is compared bit for bit with the oracle; solves to
the contract of tests/test_gpu_parity.py.  B200LDU_DRYRUN_ORACLE=1 runs the parts the stand-in tests/oracle_backend.py has
(tests/test_polymesh_cpu.py does that on a machine without a GPU)."""
import importlib
import os

import numpy as np
import pytest

import polymesh_cases as pc
from oracle import interfoam_oracle as io
from oracle import mules_oracle as mo
from test_mules_cpu import COMBOS
from test_oracle_fvm import full_system, make

pytestmark = pytest.mark.gpu


def dry():
    return os.environ.get("B200LDU_DRYRUN_ORACLE") == "1"


@pytest.fixture(scope="module")
def gpu():
    if dry():
        import oracle_backend
        yield oracle_backend.fixture()
        return
    import torch
    assert torch.cuda.is_available()
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


def box(kind):
    """the small meshes of the bit-for-bit tests"""
    if kind == "graph":
        return pc.graph(400, 4, 31)
    if kind == "periodic":
        return pc.refined_box(5, "random", periodic_x=True, seed=4)
    return pc.refined_box(6, kind, seed=2)


KINDS = list(pc.ORDERS) + ["graph"]


def _t(gpu):
    capi, ctx, torch = gpu
    return lambda a: None if a is None else torch.from_numpy(np.array(a, dtype=np.float64).ravel()).to(ctx.device)


def host(x, nc=None):
    a = x.cpu().numpy()
    return a if nc is None else a.reshape(-1, nc)


def device_addr(gpu, b):
    capi, ctx, _ = gpu
    a = capi.mesh_to_device(ctx, b)
    capi.fv_boundary_set(a, b.bFaceCells)
    return a


# ---- a. face sums (csrc/fv.cu) -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS + ["periodic"])
def test_face_sums(gpu, orc, kind):
    capi, ctx, torch = gpu
    b = box(kind)
    t = _t(gpu)
    oa = pc.addr(orc, b)
    A = device_addr(gpu, b)
    rng = np.random.default_rng(5)
    n, nF, bfc = b.nCells, b.nFaces, b.bFaceCells
    nB = len(bfc)
    V, Sf, bSf, w = b.volumes(), b.Sf(), b.bSf, b.weights()
    for nc in (1, 3):
        ssf, bssf = rng.uniform(-1, 1, (nF, nc)), rng.uniform(-1, 1, (nB, nc))
        for div in (0, 1):
            for sign in (1, -1):
                got = host(capi.fv_surface_integrate(A, nc, t(ssf), t(bssf), t(V), bool(div), sign))
                want = np.asarray(orc.surface_integrate(oa, ssf.ravel(), bfc, bssf.ravel(), V, nc, bool(div), sign)).ravel()
                assert np.array_equal(got, want), (kind, nc, div, sign)
        vf = rng.uniform(-1, 1, (n, nc))
        sf = host(capi.fv_interpolate_linear(A, nc, t(w), t(vf)))
        assert np.array_equal(sf, np.asarray(orc.interpolate_linear(oa, w, vf.ravel(), nc)).ravel()), kind
        got = host(capi.fv_grad_linear(A, nc, t(Sf), t(w), t(vf), t(bSf), t(bssf), t(V)))
        want = orc.gauss_grad(oa, Sf.ravel(), sf, bfc, bSf.ravel(), bssf.ravel(), V, nc)
        assert np.array_equal(got, np.asarray(want).ravel()), (kind, nc)
        if not dry():
            L, dp = capi.lib(), capi._dp
            keep = [t(Sf), t(ssf), t(bSf), t(bssf), t(V)]
            out = torch.empty(n * 3 * nc, dtype=torch.float64, device=ctx.device)
            capi.check(L.b200ldu_fv_gauss_grad(A.h, nc, *(dp(k) for k in keep), dp(out)))
            want = orc.gauss_grad(oa, Sf.ravel(), ssf.ravel(), bfc, bSf.ravel(), bssf.ravel(), V, nc)
            assert np.array_equal(host(out), np.asarray(want).ravel()), (kind, nc)
        delta = b.deltaCoeffs()
        got = host(capi.fv_sngrad(A, nc, t(delta), t(vf)))
        assert np.array_equal(got, np.asarray(orc.sngrad(oa, delta, vf.ravel(), nc)).ravel())
        if kind == "periodic":
            pnf = host(capi.fv_patch_neighbour_field(A, nc, t(vf)), nc)
            assert np.array_equal(pnf, vf[b.coupled_arrays()[3]])
    U = rng.uniform(-1, 1, (n, 3))
    Uf = np.asarray(orc.interpolate_linear(oa, w, U.ravel(), 3)).reshape(nF, 3)
    assert np.array_equal(host(capi.fv_flux_linear(A, t(Sf), t(w), t(U))), pc.face_flux(Uf, Sf))
    dc, g = b.deltaCoeffs(), rng.uniform(0.5, 1.5, nF) * b.magSf()
    up, dg = capi.fv_laplacian_fill(A, t(dc), t(g))
    ru, rd = orc.laplacian_fill(oa, dc, g)
    assert np.array_equal(host(up), ru) and np.array_equal(host(dg), rd)
    phi = pc.face_flux(pc.velocity(b.face_centres()), Sf)
    lw, uw, dw = capi.fv_convection_fill(A, t(w), t(phi))
    rl, ru, rd = orc.convection_fill(oa, w, phi)
    assert np.array_equal(host(lw), rl) and np.array_equal(host(uw), ru) and np.array_equal(host(dw), rd)
    if not dry():
        L, dp = capi.lib(), capi._dp
        ic, d0 = rng.uniform(-1, 1, nB), rng.uniform(1, 2, n)
        icd, dd, ss = t(ic), t(d0), t(d0)
        capi.check(L.b200ldu_fv_add_boundary_diag(A.h, dp(icd), dp(dd)))
        assert np.array_equal(host(dd), orc.add_boundary_diag(bfc, ic, d0))
        capi.check(L.b200ldu_fv_add_boundary_source(A.h, dp(icd), dp(ss)))
        assert np.array_equal(host(ss), orc.add_boundary_source(bfc, ic, d0))
    A.close()


def test_gauss_grad_of_a_linear_field_is_exact(gpu, orc):
    """independent of the oracle: the device's Gauss gradient of the face values of phi = a.x + b against the same sum in exact
    rational arithmetic (tests/polymesh_cases.check_exact_gauss_grad), and the surface integral of U.Sf for a constant U around 0"""
    capi, ctx, torch = gpu
    b = pc.refined_box(5, "random", seed=8)
    t = _t(gpu)
    A = device_addr(gpu, b)
    a_, b_ = np.array([0.7, -1.3, 2.1]), 0.4
    phif, phib = b.face_centres() @ a_ + b_, b.bCf @ a_ + b_
    V = b.volumes()
    oa = pc.addr(orc, b)
    if dry():
        got = np.asarray(orc.gauss_grad(oa, b.Sf().ravel(), phif, b.bFaceCells, b.bSf.ravel(), phib, V, 1)).reshape(-1, 3)
    else:
        L, dp = capi.lib(), capi._dp
        keep = [t(b.Sf()), t(phif), t(b.bSf), t(phib), t(V)]
        out = torch.empty(b.nCells * 3, dtype=torch.float64, device=ctx.device)
        capi.check(L.b200ldu_fv_gauss_grad(A.h, 1, *(dp(k) for k in keep), dp(out)))
        got = host(out, 3)
    pc.check_exact_gauss_grad(b, phif, phib, got, a_)
    U = np.array([0.3, -0.8, 1.1])
    got = host(capi.fv_surface_integrate(A, 1, t(b.Sf() @ U), t(b.bSf @ U), t(V), False, -1))
    pc.check_closed_sum(b, U, got)
    A.close()


# ---- b. fvMatrix glue (csrc/fvmatrix.cu) ---------------------------------------------------------------------------------
def _glue(gpu, orc, b, nc, seed):
    from test_zzz_fvm_gpu import Dev
    a, d, kw = pc.fvm_case(orc, b, nc, seed)
    x = np.random.default_rng(seed + 1).uniform(-1, 1, (b.nCells, nc))
    cou = (kw["couBou"], kw["couInt"]) if kw else None
    return a, d, kw, x, cou, Dev


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("kind", list(pc.ORDERS) + ["periodic"])
def test_fvm_operations(gpu, orc, kind, nc):
    capi, ctx, torch = gpu
    b = box(kind)
    a, d, kw, x, cou, Dev = _glue(gpu, orc, b, nc, 3)
    ofm = make(orc, a, d, nc, x, **kw)
    D = Dev(gpu, b, d, nc, x, cou=cou)
    nC = 0 if not kw else len(b.coupled_arrays()[1])
    pnf = ofm.patchNeighbourField() if nC else None
    pnf_d = D.t(pnf) if nC else None
    if nC:
        assert np.array_equal(pnf, x[b.coupled_arrays()[3]])
        assert np.array_equal(host(capi.fv_patch_neighbour_field(D.addr, nc, D.t(x)), nc), pnf)
    assert np.array_equal(host(D.fv.A()), ofm.A())
    assert np.array_equal(host(D.fv.H(pnf_d), nc), ofm.H())
    fi, fb, fcp = D.fv.flux(D.nB, nC, pnf_d)
    oi, ob, oc = ofm.flux()
    assert np.array_equal(host(fi, nc), oi) and np.array_equal(host(fb, nc), ob) and np.array_equal(host(fcp, nc), oc)
    for cmpt in list(range(nc)) + [-1]:
        got = D.t(d["diag"])
        D.fv.addBoundaryDiag(got, cmpt) if cmpt >= 0 else D.fv.addCmptAvBoundaryDiag(got)
        ref = d["diag"].copy()
        ofm.addBoundaryDiag(ref, cmpt) if cmpt >= 0 else ofm.addCmptAvBoundaryDiag(ref)
        assert np.array_equal(host(got), ref), cmpt
    for couples in ((False, True) if nC else (False,)):
        src = D.t(d["source"])
        D.fv.addBoundarySource(src, pnf_d if couples else None)
        ref = np.array(d["source"], float).reshape(b.nCells, nc).copy()
        ofm.addBoundarySource(ref, couples)
        assert np.array_equal(host(src, nc), ref), couples
    if nc == 1:
        got, want = host(D.fv.residual(pnf_d)), ofm.residual()
        if nC:    # the doubled neighbour term of a coupled residual: rounding apart (tests/test_zzz_fvm_gpu.py)
            np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-14 * np.abs(want).max())
        else:
            assert np.array_equal(got, want)
    for alpha in (1.0, 0.7):
        Dr = Dev(gpu, b, d, nc, x, addr=D.addr, cou=cou)
        orl = make(orc, a, d, nc, x, **kw)
        Dr.fv.relax(alpha)
        orl.relax(alpha)
        assert np.array_equal(host(Dr.diag), orl.diag) and np.array_equal(host(Dr.source, nc), orl.source), alpha
        Dr.mat.close()
    val = [0.5, -1.25, 2.0][:nc]
    D.fv.setReference(11, val)
    ofm.setReference(11, val)
    assert np.array_equal(host(D.diag), ofm.diag) and np.array_equal(host(D.source, nc), ofm.source)
    D.close()


@pytest.mark.parametrize("nc,solver,pre", [(1, "PCG", "DIC"), (3, "PBiCG", "DILU"), (1, "GAMG", "GaussSeidel")])
@pytest.mark.parametrize("kind", ["coarse-first", "random", "periodic"])
def test_fvm_solve(gpu, orc, kind, nc, solver, pre):
    """fvm_solve against a dense numpy solve of the folded system (1e-8) and the oracle's solve (counts within 2, initial
    residual 1e-10)"""
    capi = gpu[0]
    b = box(kind)
    a, d, kw, _, cou, Dev = _glue(gpu, orc, b, nc, 4)
    ctl = dict(tolerance=1e-11, maxIter=1000)
    z = np.zeros((b.nCells, nc))
    oz = make(orc, a, d, nc, z, **kw)
    pnf = oz.patchNeighbourField() if kw else None
    D = Dev(gpu, b, d, nc, z, cou=cou)
    gg = og = None
    if solver == "GAMG":
        gg = capi.GamgAgglomeration(D.addr, b.magSf(), 10, 1)
        og = orc.Gamg(a, b.magSf(), 10, 1)
    psi_ref, perfs_ref, _ = oz.solve(solver, pre, og, pnf, **ctl)
    perfs = D.fv.solve(solver, pre, gamg=gg, pnf=D.t(pnf) if kw else None, **ctl)
    for k in range(nc):
        assert perfs[k].converged and perfs_ref[k].converged
        assert abs(perfs[k].nIterations - perfs_ref[k].nIterations) <= (0 if solver == "GAMG" else 2), \
            (k, perfs[k].nIterations, perfs_ref[k].nIterations)
        np.testing.assert_allclose(perfs[k].initialResidual, perfs_ref[k].initialResidual, rtol=1e-10)
    psi = host(D.psi, nc)
    np.testing.assert_allclose(psi, psi_ref, rtol=0, atol=1e-8)
    if not kw:
        for k in range(nc):
            Ad, rhs = full_system(b, d, k)
            np.testing.assert_allclose(psi[:, k], np.linalg.solve(Ad, rhs), rtol=0, atol=1e-8)
    if gg is not None:
        gg.close()
    D.close()


# ---- c. LduCoeffs (csrc/lduops.cu) ---------------------------------------------------------------------------------------
LDU_KINDS = {"diagonal": ("diag",), "symmetric": ("diag", "upper"), "asymmetric": ("diag", "upper", "lower"), "empty": ()}


def _mat(b, kind, seed):
    """the arrays of one kind of lduMatrix (tests/test_lduops.py)"""
    rng = np.random.default_rng(seed)
    full = dict(diag=rng.uniform(1, 2, b.nCells), upper=rng.uniform(-1, 1, b.nFaces), lower=rng.uniform(-1, 1, b.nFaces))
    return {k: full[k] for k in LDU_KINDS[kind]}


@pytest.mark.parametrize("kind", ["fine-first", "graph"])
def test_ldu_algebra(gpu, orc, kind):
    import itertools
    from oracle import lduops_oracle as lop
    if dry():
        pytest.skip("the stand-in has no LduCoeffs")
    capi, ctx, torch = gpu
    b = box(kind)
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(ctx.device)
    A_ = capi.mesh_to_device(ctx, b)
    for ka, kb, sub in itertools.product(["diagonal", "symmetric", "asymmetric", "empty"], ["diagonal", "symmetric", "asymmetric"],
                                         [False, True]):
        A, B = _mat(b, ka, 3), _mat(b, kb, 4)
        dA = capi.LduCoeffs(A_, t(A.get("diag")), t(A.get("upper")), t(A.get("lower")))
        dB = capi.LduCoeffs(A_, t(B.get("diag")), t(B.get("upper")), t(B.get("lower")))
        if sub:
            dA -= dB
        else:
            dA += dB
        want = lop.add_assign(A, B, b.nCells, sub)
        got = dict(zip(("diag", "upper", "lower"), (None if x is None else host(x) for x in dA.arrays())))
        assert sorted(k for k, v in got.items() if v is not None) == sorted(want), (ka, kb, sub)
        for k, v in want.items():
            assert np.array_equal(got[k], v), (ka, kb, sub, k)
    A = _mat(b, "asymmetric", 5)
    sf = np.random.default_rng(6).uniform(0.5, 2, b.nCells)
    for s in (sf, 1.7):
        dd = capi.LduCoeffs(A_, t(A["diag"]), t(A["upper"]), t(A["lower"]))
        dd.scale(t(s) if not np.isscalar(s) else s)
        want = lop.scale(A, s, b.lower, b.upper)
        for k, v in zip(("diag", "upper", "lower"), dd.arrays()):
            assert np.array_equal(host(v), want[k]), k
    oa = orc.Addr(b.nCells, b.lower, b.upper)
    for kd in ("symmetric", "asymmetric"):
        A = _mat(b, kd, 7)
        dd = capi.LduCoeffs(A_, t(A["diag"]), t(A["upper"]), t(A.get("lower")))
        for mode, fn in ((0, "orc_sumDiag"), (1, "orc_negSumDiag"), (2, "orc_sumMagOffDiag")):
            ref = A["diag"].copy()
            low = A.get("lower")
            getattr(orc.lib(), fn)(oa.h, orc._d(A["upper"]), orc._d(low) if low is not None else None, orc._d(ref))
            assert np.array_equal(host(dd.row_sum(mode, t(A["diag"].copy()))), ref), (kd, mode)
    A_.close()


# ---- d. limited schemes and the interface flux (csrc/fieldops.cu, csrc/vof.cu) -----------------------------------------
@pytest.mark.parametrize("kind", list(pc.ORDERS))
def test_limited_flux_and_interface_flux(gpu, orc, kind):
    if dry():
        pytest.skip("the stand-in has no limiter, limited-flux or interface-flux entry points")
    capi, ctx, torch = gpu
    b = box(kind)
    t = _t(gpu)
    A = device_addr(gpu, b)
    ops = capi.FieldOps(ctx)
    oa = pc.addr(orc, b)
    rng = np.random.default_rng(41)
    C = b.cell_centres()
    vf = np.sin(3 * C[:, 0]) * np.cos(2 * C[:, 1]) + C[:, 2]
    vf[rng.uniform(0, 1, b.nCells) < 0.1] = 0.25
    vfB = np.sin(3 * b.bCf[:, 0]) * np.cos(2 * b.bCf[:, 1]) + b.bCf[:, 2]
    sf = host(capi.fv_interpolate_linear(A, 1, t(b.weights()), t(vf)))
    gradc = np.asarray(orc.gauss_grad(oa, b.Sf().ravel(), sf, b.bFaceCells, b.bSf.ravel(), vfB, b.volumes(), 1)).reshape(-1, 3)
    flux = pc.face_flux(pc.velocity(b.face_centres()), b.Sf())
    flux[::11] = 0.0
    cd = b.weights()
    for scheme, ks in (("upwind", (1.0,)), ("linear", (1.0,)), ("limitedLinear", (1.0, 0.5)), ("vanLeer", (1.0,)), ("Minmod", (1.0,))):
        for k in ks:
            for fs, os_ in ((1, 1), (-1, -1), (-1, 1), (1, -1)):
                got = host(capi.fv_limited_flux(A, scheme, t(flux), t(vf), t(gradc), t(C), t(cd), k, fs, os_))
                want = io.limited_flux(scheme, b.lower, b.upper, flux, vf, gradc, C, cd, k, fs, os_)
                assert np.array_equal(got, want), (scheme, k, fs, os_)
                F = ops.neg(t(flux)) if fs < 0 else t(flux)
                w = capi.fv_limited_weights(ctx, F, capi.fv_limiter(A, scheme, F, t(vf), t(gradc), t(C), k), t(cd))
                comp = ops.mul(F, capi.fv_interpolate_linear(A, 1, w, t(vf)))
                assert np.array_equal(got, host(ops.neg(comp) if os_ < 0 else comp)), (scheme, k, fs, os_)
    bSn = rng.uniform(-1, 1, len(b.bFaceCells))
    bSn[::3] = 0.0
    g = rng.uniform(-1, 1, (b.nCells, 3))
    g[rng.uniform(0, 1, b.nCells) < 0.3] = 0.0
    for deltaN in (1e-8, 0.5):
        for withPhi in (False, True):
            nHatf, nHatfB, phir = capi.vof_interface_flux(A, t(b.weights()), t(g), t(b.Sf()), t(b.bSf), t(bSn), deltaN,
                                                          t(flux) if withPhi else None, t(b.magSf()) if withPhi else None, 0.75)
            w0, w1, w2 = io.interface_flux(b.lower, b.upper, b.weights(), g, b.Sf(), b.bFaceCells, b.bSf, bSn, deltaN,
                                           flux if withPhi else None, b.magSf(), 0.75)
            assert np.array_equal(host(nHatf), w0) and np.array_equal(host(nHatfB), w1), (deltaN, withPhi)
            assert (phir is None) if not withPhi else np.array_equal(host(phir), w2)
    # independent of the oracle: the exact gradient of a linear alpha gives nHatf = a/(|a| + deltaN).Sf within a few ulps
    a_ = np.array([0.3, -0.5, 0.8])
    deltaN = 1e-8
    nHatf, _, _ = capi.vof_interface_flux(A, t(b.weights()), t(np.tile(a_, (b.nCells, 1))), t(b.Sf()), t(b.bSf), t(bSn), deltaN)
    pc.check_interface_normal(b, a_, deltaN, host(nHatf))
    A.close()


# ---- e. MULES (csrc/mules.cu, rapidcfd-dev_b200/mules.py) ----------------------------------------------------------------
@pytest.mark.parametrize("combo", COMBOS)
@pytest.mark.parametrize("kind", KINDS)
def test_mules(gpu, kind, combo):
    capi, ctx, torch = gpu
    mules = importlib.import_module("rapidcfd-dev_b200.mules")
    b = box(kind)
    d = pc.mules_case(b, 12, combo)
    kw = d["kw"]
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(ctx.device)
    A = device_addr(gpu, b)
    ops = capi.FieldOps(ctx)
    tk = {k: t(v) for k, v in kw.items()}
    L, U, bfc = b.lower, b.upper, d["bfc"]
    bd, bdB = mo.upwind_flux(L, U, d["phi"], d["phiB"], d["psi"], d["psiB"])
    corr, corrB = d["phiPsi"] - bd, d["phiPsiB"] - bdB
    for nIter in (0, 1, 3):
        lam, lamB = capi.mules_limiter(A, t(d["V"]), d["rDeltaT"], t(d["psi"]), t(d["psi0"]), t(d["psiB"]), t(bd), t(bdB), t(corr),
                                       t(corrB), 1.0, 0.0, nIter, tk.get("rho"), tk.get("rho0"), tk.get("Sp"), tk.get("Su"))
        want, wantB = mo.limiter(d["n"], L, U, bfc, d["V"], d["rDeltaT"], d["psi"], d["psi0"], d["psiB"], bd, bdB, corr, corrB,
                                 1.0, 0.0, nIter, **kw)
        assert np.array_equal(host(lam), want) and np.array_equal(host(lamB), wantB), nIter
        assert nIter == 0 or (want < 1).sum() > d["nF"] // 10          # the limiter is active on this case
    kc = {k: v for k, v in kw.items() if k != "rho0"}
    cB = corrB + 1e-5 * np.sin(np.arange(d["nB"]))
    for ex in (0.0, 0.2):
        lam, lamB = capi.mules_limiter_corr(A, t(d["V"]), d["rDeltaT"], t(d["psi"]), t(d["psiB"]), t(d["phiB"]), t(corr), t(cB), 1.0, 0.0, 3,
                                            tk.get("rho"), tk.get("Sp"), tk.get("Su"), ex)
        want, wantB = mo.limiter(d["n"], L, U, bfc, d["V"], d["rDeltaT"], d["psi"], d["psi"], d["psiB"], np.zeros(d["nF"]), d["phiB"],
                                 corr, cB, 1.0, 0.0, 3, kc.get("rho"), None, kc.get("Sp"), kc.get("Su"), corr=True, extremaCoeff=ex)
        assert np.array_equal(host(lam), want) and np.array_equal(host(lamB), wantB), ex
    lp, lpB = mules.limit(capi, A, ops, t(d["V"]), d["rDeltaT"], t(d["psi"]), t(d["psi0"]), t(d["psiB"]), t(d["phi"]), t(d["phiB"]),
                          t(d["phiPsi"]), t(d["phiPsiB"]), 1.0, 0.0, 3, **tk)
    want, wantB = mo.limit(d["n"], L, U, bfc, d["V"], d["rDeltaT"], d["psi"], d["psi0"], d["psiB"], d["phi"], d["phiB"], d["phiPsi"],
                           d["phiPsiB"], 1.0, 0.0, 3, **kw)
    assert np.array_equal(host(lp), want) and np.array_equal(host(lpB), wantB)
    new = mules.explicit_solve(capi, A, ops, t(d["V"]), d["rDeltaT"], t(d["psi0"]), lp, lpB, **tk)
    assert np.array_equal(host(new), mo.explicit_solve(d["n"], L, U, bfc, d["V"], d["rDeltaT"], d["psi0"], want, wantB, **kw))
    tkc = {k: v for k, v in tk.items() if k != "rho0"}
    lc, lcB = mules.limit_corr(capi, A, ops, t(d["V"]), d["rDeltaT"], t(d["psi"]), t(d["psiB"]), t(d["phiB"]), t(corr), t(cB), 1.0, 0.0,
                               3, **tkc)
    want, wantB = mo.limit_corr(d["n"], L, U, bfc, d["V"], d["rDeltaT"], d["psi"], d["psiB"], d["phiB"], corr, cB, 1.0, 0.0, 3, **kc)
    assert np.array_equal(host(lc), want) and np.array_equal(host(lcB), wantB)
    new = mules.correct(capi, A, ops, t(d["V"]), d["rDeltaT"], t(d["psi"]), lc, lcB, **tkc)
    assert np.array_equal(host(new), mo.correct(d["n"], L, U, bfc, d["V"], d["rDeltaT"], d["psi"], want, wantB, **kc))
    A.close()


def test_mules_step_is_bounded_and_conservative(gpu):
    """independent of the oracle: explicit MULES steps of a rotating U on the split-hex box (tests/polymesh_cases.mules_rotation)"""
    capi, ctx, torch = gpu
    mules = importlib.import_module("rapidcfd-dev_b200.mules")
    b = pc.refined_box(8, "random", seed=3)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(ctx.device)
    A = device_addr(gpu, b)
    ops = capi.FieldOps(ctx)

    def step(psi, phi, phiB, psiB, dt, limited):
        p = t(psi)
        phiPsi = host(ops.mul(t(phi), capi.fv_interpolate_linear(A, 1, t(b.weights()), p)))
        phiPsiB = phiB * psiB
        if limited:
            lp, lpB = mules.limit(capi, A, ops, t(b.volumes()), 1 / dt, p, p, t(psiB), t(phi), t(phiB), t(phiPsi), t(phiPsiB), 1.0, 0.0, 3)
        else:
            lp, lpB = t(phiPsi), t(phiPsiB)
        return host(mules.explicit_solve(capi, A, ops, t(b.volumes()), 1 / dt, t(psi), lp, lpB)), host(lpB)
    pc.check_mules_rotation(b, step)
    A.close()


# ---- f. engine: asymmetric matrices, bands, streams ----------------------------------------------------------------------
ENGINE = [pytest.param("box21", band, id=f"box21-{band}") for band in (64, 512, 2048)] + [pytest.param("random30000", 16384, id="random30000")]


@pytest.fixture(scope="module")
def engine_problems(orc):
    cache = {}

    def get(name):
        if name not in cache:
            if name == "box21":
                b = pc.refined_box(21, "random", seed=5)
                a, diag, up, low = pc.asym_matrix(orc, b)
                cache[name] = (b, b.nCells, b.lower, b.upper, b.cell_centres(), diag, up, low)
            else:
                from test_layout_cpu import _RandomGraph
                g = _RandomGraph(30000, 4, 1)
                rng = np.random.default_rng(17)
                up, low = rng.uniform(-1.0, 1.0, g.nFaces), rng.uniform(-1.0, 1.0, g.nFaces)
                s = np.zeros(g.nCells)
                np.add.at(s, g.lower, np.abs(up) + np.abs(low))
                np.add.at(s, g.upper, np.abs(up) + np.abs(low))
                diag = -(s + 0.1) * rng.uniform(1.0, 1.5, g.nCells)
                cache[name] = (None, g.nCells, np.asarray(g.lower, np.int32), np.asarray(g.upper, np.int32), None, diag, up, low)
        return cache[name]
    return get


def _asym_ops(mat, t, x, b):
    out = {"Amul": mat.Amul(t(x)), "Tmul": mat.Tmul(t(x)), "residual": mat.residual(t(x), t(b)), "H": mat.H(t(x)),
           "faceH": mat.faceH(t(x)), "sumA": mat.sumA(t(x)), "H1": mat.H1(t(x))}
    for pre in ("none", "diagonal", "DILU"):
        for T in (False, True):
            out[f"precondition-{pre}-T{int(T)}"] = mat.precondition(pre, t(x), T)
    for ns in (1, 2, 3):
        out[f"GaussSeidel-{ns}"] = mat.smooth("GaussSeidel", t(x), t(b), ns)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _asym_ref(om, x, b):
    ref = {"Amul": om.amul(x), "Tmul": om.tmul(x), "residual": om.residual(x, b), "H": om.H(x), "faceH": om.faceH(x),
           "sumA": om.sumA(), "H1": om.H1()}
    for pre in ("none", "diagonal", "DILU"):
        for T in (False, True):
            ref[f"precondition-{pre}-T{int(T)}"] = om.precondition(pre, x, T)
    for ns in (1, 2, 3):
        ref[f"GaussSeidel-{ns}"] = om.jacobi(x, b, ns)
    return ref


def _compare_ops(M, got, ref, what, coupled=False):
    for op, r in ref.items():
        if op.startswith("precondition-DILU") or (coupled and op.startswith("GaussSeidel")):
            M.close(got[op], r, f"{op} [{what}]", 1e-13)      # AINV's association; Jacobi with coupled interfaces (DESIGN.md 2)
        else:
            M.bits_es(got[op], r, f"{op} [{what}]")


@pytest.mark.parametrize("name,band", ENGINE)
def test_engine_asymmetric(gpu, orc, engine_problems, name, band):
    """every row-gather operation of an asymmetric matrix (entry stream) at several band sizes, bit for bit the oracle except the
    stated exceptions, on the three input families of tests/test_gpu_engine_streams.py; Amul, Tmul and residual also against
    long-double products (tests/polymesh_cases.check_matrix_products)"""
    from test_gpu_engine_streams import Mismatches, Problem, engine_env
    if dry():
        pytest.skip("band sizes and streams are the device layout's")
    capi, ctx, torch = gpu
    b, n, L, U, C, diag, up, low = engine_problems(name)
    with engine_env(band, None):
        A = capi.LduAddressing(ctx, n, L, U, cellCentres=C)
    assert A.info()["nBands"] > 1      # an asymmetric matrix runs on the entry stream whatever the layout offers
    mat = capi.LduMatrix(A)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(ctx.device)
    keep = (t(diag), t(up), t(low))
    mat.set(*keep)
    oa = orc.Addr(n, L, U)
    om = orc.Matrix(oa, diag, up, low)
    pb = Problem(orc, n, L, U, diag, up, seed=3)
    M = Mismatches()
    for inp, x, rhs in (("field", pb.field(3), pb.field(4)), ("signed-zeros", pb.signed_zeros(5), pb.signed_zeros(6)),
                        ("wide", pb.wide(7), pb.wide(8))):
        got = _asym_ops(mat, t, x, rhs)
        _compare_ops(M, got, _asym_ref(om, x, rhs), inp)
        if inp == "field":
            pc.check_matrix_products(M, L, U, diag, up, low, x, rhs, got)
    M.check()
    mat.close()
    A.close()


def test_engine_asymmetric_cyclic(gpu, orc):
    """an asymmetric matrix with the cyclic pair (four coupled faces per unsplit cell) and distinct bou / int arrays"""
    from test_gpu_engine_streams import Mismatches
    capi, ctx, torch = gpu
    if dry():
        pytest.skip("band sizes and streams are the device layout's")
    b = box("periodic")
    a, d, kw = pc.fvm_case(orc, b, 3, 9)
    ps, fc, nr, _ = b.coupled_arrays()
    A = capi.LduAddressing(ctx, b.nCells, b.lower, b.upper, ps, fc, nr, b.cell_centres())
    mat = capi.LduMatrix(A)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(ctx.device)
    keep = (t(d["diag"]), t(d["upper"]), t(d["lower"]), t(kw["couBou"]), t(kw["couInt"]))
    mat.set(*keep)
    om = orc.Matrix(a, d["diag"], d["upper"], d["lower"], kw["couBou"], kw["couInt"])
    rng = np.random.default_rng(2)
    x, rhs = rng.uniform(-1, 1, b.nCells), rng.uniform(-1, 1, b.nCells)
    M = Mismatches()
    got = _asym_ops(mat, t, x, rhs)
    _compare_ops(M, got, _asym_ref(om, x, rhs), "cyclic", coupled=True)
    M.check()
    mat.close()
    A.close()


@pytest.mark.parametrize("band", [64, 512])
def test_engine_symmetric_streams(gpu, orc, band):
    """a symmetric matrix on the split-hex box: face stream against entry stream bit for bit, both against the oracle"""
    from test_gpu_engine_streams import Mismatches, Problem, _ops, _ops_oracle, engine_env
    if dry():
        pytest.skip("band sizes and streams are the device layout's")
    capi, ctx, torch = gpu
    b = pc.refined_box(12, "fine-first")
    a, diag, up = pc.sym_matrix(orc, b)
    pb = Problem(orc, b.nCells, b.lower, b.upper, diag, up, b.cell_centres(), seed=4)

    class Side:
        def __init__(self, fs):
            with engine_env(band, fs):
                self.addr = capi.LduAddressing(ctx, b.nCells, b.lower, b.upper, cellCentres=b.cell_centres())
            self.info, self.mat, self.pb = self.addr.info(), capi.LduMatrix(self.addr), pb
            self.keep = (self.t(diag), self.t(up))
            self.mat.set(*self.keep)

        def t(self, v):
            return torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(ctx.device)

    es, fs = Side(0), Side(1)
    assert not es.info["faceStream"] and fs.info["faceStream"] and fs.info["nBands"] > 1
    M = Mismatches()
    for inp, x, rhs in (("field", pb.field(3), pb.field(4)), ("signed-zeros", pb.signed_zeros(5), pb.signed_zeros(6)),
                        ("wide", pb.wide(7), pb.wide(8))):
        ge, gf = _ops(es, x, rhs), _ops(fs, x, rhs)
        ref = _ops_oracle(pb.om, x, rhs, False)
        for op, v in gf.items():
            M.bits_es(ge[op], v, f"{op} [{inp}] ES vs FS")
            if op.startswith("precondition-DIC"):
                M.close(v, ref[op], f"{op} [{inp}] FS vs oracle", 1e-13)
            else:
                M.bits(v, ref[op], f"{op} [{inp}] FS vs oracle")
    M.check()
    for s in (es, fs):
        s.mat.close()
        s.addr.close()


# ---- g. solvers ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def solver_box(gpu, orc):
    capi, ctx, torch = gpu
    b = pc.refined_box(10, "random", seed=6)
    A = capi.LduAddressing(ctx, b.nCells, b.lower, b.upper, cellCentres=b.cell_centres())
    yield b, A
    A.close()


@pytest.mark.parametrize("solver,pre", [(s, p) for s in ("PBiCG", "PBiCGStab") for p in ("DILU", "diagonal", "none")] +
                         [("smoothSolver", "GaussSeidel"), ("PCG", "DIC"), ("PCG", "none")])
def test_solvers(gpu, orc, solver_box, solver, pre):
    from test_gpu_parity import _cmp_hist
    capi, ctx, torch = gpu
    b, A = solver_box
    sym = solver == "PCG"
    a, diag, up, low = pc.asym_matrix(orc, b) if not sym else pc.sym_matrix(orc, b) + (None,)
    om = orc.Matrix(a, diag, up, low)
    t = lambda v: None if v is None else torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(ctx.device)
    mat = capi.LduMatrix(A)
    keep = (t(diag), t(up), t(low))
    mat.set(*keep)
    xs = np.random.default_rng(42).uniform(-1, 1, b.nCells)
    rhs = om.amul(xs)
    smooth = solver == "smoothSolver"
    ctl = dict(tolerance=1e-8, maxIter=300) if not smooth else dict(tolerance=1e-6, maxIter=300, nSweeps=2)
    psi_ref, pr, href = om.solve(solver, pre, np.zeros(b.nCells), rhs, **ctl)
    psi = torch.zeros(b.nCells, dtype=torch.float64, device=ctx.device)
    perf, hist = mat.solve(solver, pre, psi, t(rhs), histCap=1024, **ctl)
    assert perf.solverName == pr.solverName and perf.converged == pr.converged == 1
    assert abs(perf.nIterations - pr.nIterations) <= (0 if pr.nIterations < 100 else 1), (perf.nIterations, pr.nIterations)
    # the bi-conjugate recurrences amplify the different order of the global sums once the residual is small: measured on an
    # H100 80GB HBM3 (700 W limit) 6e-16 absolute (3e-8 relative) at a residual of 4e-8 for PBiCGStab without preconditioner, so
    # 1e-9 relative above a residual of 1e-6 and 1e-15 absolute below
    _cmp_hist(hist, href, first=30, rtol=1e-9, floor=0.0 if (sym or smooth) else 1e-6)
    np.testing.assert_allclose(host(psi), psi_ref, rtol=0, atol=1e-6)
    mat.close()


@pytest.mark.parametrize("merge", [1, 2])
@pytest.mark.parametrize("kind", ["symmetric", "asymmetric"])
def test_gamg(gpu, orc, solver_box, kind, merge):
    """agglomeration maps identical to the oracle's on every level (face weights |Sf|), cycle counts identical, history to 1e-8"""
    capi, ctx, torch = gpu
    b, A = solver_box
    a, diag, up, low = pc.asym_matrix(orc, b) if kind == "asymmetric" else pc.sym_matrix(orc, b) + (None,)
    om = orc.Matrix(a, diag, up, low)
    w = b.magSf()
    og = orc.Gamg(a, w, 10, mergeLevels=merge)
    gg = capi.GamgAgglomeration(A, w, 10, mergeLevels=merge)
    assert gg.nLevels == og.nLevels and gg.nLevels >= 3
    for lev in range(gg.nLevels):
        assert np.array_equal(gg.restrict_addr(lev), og.restrict_addr(lev)), lev
    t = lambda v: None if v is None else torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(ctx.device)
    mat = capi.LduMatrix(A)
    keep = (t(diag), t(up), t(low))
    mat.set(*keep)
    rhs = om.amul(np.random.default_rng(43).uniform(-1, 1, b.nCells))
    ctl = dict(tolerance=1e-9, maxIter=100)
    psi_ref, pr, href = og.solve(om, "GaussSeidel", np.zeros(b.nCells), rhs, **ctl)
    psi = torch.zeros(b.nCells, dtype=torch.float64, device=ctx.device)
    perf, hist = mat.solve("GAMG", "GaussSeidel", psi, t(rhs), gamg=gg, histCap=512, **ctl)
    assert perf.converged and perf.nIterations == pr.nIterations, (perf.nIterations, pr.nIterations)
    # cycle residuals within 1e-8 relative, or 1e-15 absolute (normalised) where they fall below 1e-7: the global sums' order
    # differs, measured on an H100 80GB HBM3 (700 W limit) 2.6e-16 absolute at a residual of 2.5e-9
    np.testing.assert_allclose(hist, href, rtol=1e-8, atol=1e-15)
    np.testing.assert_allclose(host(psi), psi_ref, rtol=0, atol=1e-8)
    gg.close()
    mat.close()
