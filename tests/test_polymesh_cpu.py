"""The split-hex polyhedral meshes of tests/polymesh_cases.py without a GPU: the generator's invariants, the device bodies of the
cell-walking kernels executed on the host against the oracle on every cell order (bit for bit), the independent references of
tests/test_gpu_polymesh.py evaluated on the oracle's outputs, and a dry run of that module over the oracle-backed stand-in."""
import ctypes as C
import importlib

import numpy as np
import pytest

import polymesh_cases as pc
from oracle import interfoam_oracle as io
from oracle import limiters_oracle as lo
from oracle import mules_oracle as mo
from test_host_kernels_cpu import Host, _d, hk, run_all  # noqa: F401  (hk: fixture, the host build of the kernels)
from test_interfoam_cpu import _fields, hkv  # noqa: F401  (hkv: fixture, the host build of vof_kernels.cuh)
from test_oracle_fvm import full_system

ff = importlib.import_module("rapidcfd-dev_b200.foamfile")


@pytest.fixture(scope="module", params=pc.ORDERS)
def rbox(request):
    return pc.refined_box(4, request.param, seed=1)


# ---- generator invariants ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("periodic", [False, True])
def test_cells_are_closed_and_volumes_exact(periodic):
    n = 5
    b = pc.refined_box(n, "random", periodic_x=periodic, seed=3)
    pm = b.pm
    geo = pm.fv_geometry()
    S, mag = np.zeros((b.nCells, 3)), np.zeros(b.nCells)
    nI = pm.nInternalFaces
    np.add.at(S, pm.owner, geo["Sf"])
    np.add.at(S, pm.neighbour, -geo["Sf"][:nI])
    np.add.at(mag, pm.owner, geo["magSf"])
    np.add.at(mag, pm.neighbour, geo["magSf"][:nI])
    assert (np.abs(S).max(1) <= 1e-14 * mag).all()
    V = b.volumes()
    assert abs(V.sum() - 1.0) <= 1e-13
    h = 1.0 / n
    np.testing.assert_allclose(V[b.isUnsplit], h ** 3, rtol=1e-14)
    np.testing.assert_allclose(V[~b.isUnsplit], (h / 2) ** 3, rtol=1e-14)
    assert b.isUnsplit.sum() == (n ** 3 + 1) // 2 and b.nCells == b.isUnsplit.sum() + 8 * (n ** 3 // 2)
    # the coupled partner of every cyclic face is its mirror image across the box
    ps, fc, nr, partner = b.coupled_arrays()
    if periodic:
        C_ = b.cell_centres()
        np.testing.assert_allclose(np.abs(C_[fc, 0] - C_[partner, 0]), np.where(b.isUnsplit[fc], 1 - h, 1 - h / 2), rtol=0, atol=1e-14)
        np.testing.assert_allclose(C_[fc, 1:], C_[partner, 1:], rtol=0, atol=1e-14)


def test_round_trip_through_the_polymesh_files(tmp_path):
    b = pc.refined_box(4, "fine-first", periodic_x=False)
    for binary in (False, True):
        d = str(tmp_path / f"polyMesh{int(binary)}")
        ff.write_poly_mesh(d, b.pm, binary=binary)
        pm = ff.read_poly_mesh(d)
        for k in ("owner", "neighbour", "points", "faceOffsets", "faceLabels"):
            assert np.array_equal(getattr(pm, k), getattr(b.pm, k)), k
        assert [(p.name, p.type, p.nFaces, p.startFace) for p in pm.patches] == \
               [(p.name, p.type, p.nFaces, p.startFace) for p in b.pm.patches]
        r = pc.from_poly_mesh(pm)
        for k in ("cell_centres", "volumes", "Sf", "weights", "deltaCoeffs"):
            assert np.array_equal(getattr(r, k)(), getattr(b, k)()), k


def test_generators_reach_what_they_promise():
    for order in pc.ORDERS:
        k = pc.refined_box(6, order, seed=2).counts()
        big = max(k["owner"].max(), k["losort"].max())
        assert min(k["owner"].max(), k["losort"].max()) > 3 and big >= (12 if order == "random" else 24), order
        assert k["boundary"].max() == 6 and k["multiPatchCells"] > 0
    k = pc.refined_box(5, "random", periodic_x=True).counts()
    assert k["coupled"].max() == 4
    assert pc.refined_box(4, "coarse-first", split_boundary=False).counts()["boundary"].max() == 3
    g = pc.graph(400, 4, 31)
    k = g.counts()
    assert k["owner"].max() >= 10 and k["losort"].max() >= 10 and ((k["owner"] + k["losort"]) == 0).sum() >= 7


# ---- device bodies on the host -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [1, 3])
def test_face_sum_bodies(hk, orc, rbox, nc):  # noqa: F811
    b = rbox
    rng = np.random.default_rng(7)
    n, nF, bfc = b.nCells, b.nFaces, b.bFaceCells
    nB = len(bfc)
    a = orc.Addr(n, b.lower, b.upper)
    H = Host(a, dict(bfc=bfc, diag=np.zeros(n), upper=np.zeros(nF), lower=None))
    f = lambda x: np.ascontiguousarray(x, np.float64)
    ssf, bssf, V = f(rng.uniform(-1, 1, (nF, nc))), f(rng.uniform(-1, 1, (nB, nc))), f(b.volumes())
    Sf, bSf, w, vf = f(b.Sf()), f(b.bSf), f(b.weights()), f(rng.uniform(-1, 1, (n, nc)))
    hk.hk_surface_integrate.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_int]
    for div, sign in ((1, -1), (0, 1), (0, -1), (1, 1)):
        out = np.zeros((n, nc))
        hk.hk_surface_integrate(H.p(), nc, _d(ssf), _d(bssf), _d(V), _d(out), div, sign)
        want = np.asarray(orc.surface_integrate(a, ssf.ravel(), bfc, bssf.ravel(), V, nc, bool(div), sign)).reshape(n, nc)
        assert np.array_equal(out, want), (div, sign)
    hk.hk_gauss_grad.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 6
    out = np.zeros((n, 3 * nc))
    hk.hk_gauss_grad(H.p(), nc, _d(Sf), _d(ssf), _d(bSf), _d(bssf), _d(V), _d(out))
    assert np.array_equal(out, np.asarray(orc.gauss_grad(a, Sf.ravel(), ssf.ravel(), bfc, bSf.ravel(), bssf.ravel(), V, nc)).reshape(n, -1))
    hk.hk_grad_linear.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 7
    out = np.zeros((n, 3 * nc))
    hk.hk_grad_linear(H.p(), nc, _d(Sf), _d(w), _d(vf), _d(bSf), _d(bssf), _d(V), _d(out))
    face = np.asarray(orc.interpolate_linear(a, w, vf.ravel(), nc))
    assert np.array_equal(out, np.asarray(orc.gauss_grad(a, Sf.ravel(), face.ravel(), bfc, bSf.ravel(), bssf.ravel(), V, nc)).reshape(n, -1))
    up, dg = (np.ascontiguousarray(x) for x in orc.laplacian_fill(a, b.deltaCoeffs(), b.magSf()))
    hk.hk_neg_sum_diag.argtypes = [C.c_void_p] * 4
    out = np.zeros(n)
    hk.hk_neg_sum_diag(H.p(), _d(up), _d(up), _d(out))
    assert np.array_equal(out, dg)
    lw, uw, dw = (np.ascontiguousarray(x) for x in orc.convection_fill(a, w, pc.face_flux(pc.velocity(b.face_centres()), b.Sf())))
    hk.hk_neg_sum_diag(H.p(), _d(uw), _d(lw), _d(out))
    assert np.array_equal(out, dw)


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("periodic", [False, True])
def test_fvmatrix_bodies(hk, orc, nc, periodic):  # noqa: F811
    for order in pc.ORDERS:
        b = pc.refined_box(5, order, periodic_x=periodic, seed=4) if periodic else pc.refined_box(4, order, seed=4)
        a, d, kw = pc.fvm_case(orc, b, nc, 5)
        x = np.random.default_rng(6).uniform(-1, 1, (b.nCells, nc))
        if kw:
            run_all(hk, orc, a, d, nc, x, cfc=b.coupled_arrays()[1], couInt=kw["couInt"], couBou=kw["couBou"])
        else:
            run_all(hk, orc, a, d, nc, x)


def _limiter_call(hk, H, nIter, rDeltaT, A, lam, lamB, n, corr, ex):  # noqa: F811
    hk.hk_mules_limiter.argtypes = [C.c_void_p, C.c_int, C.c_double] + [C.c_void_p] * 12 + [C.c_double, C.c_double] + [C.c_void_p] * 3 + \
                                   [C.c_int, C.c_int, C.c_double]
    hk.hk_mules_limiter(H.p(), nIter, rDeltaT, _d(A["rho"]), _d(A.get("rho0")), _d(A["psi"]), _d(A["psi0"]), _d(A["psiB"]),
                        _d(A.get("bd")), _d(A["bdB"]), _d(A["corr"]), _d(A["corrB"]), _d(A["Sp"]), _d(A["Su"]), _d(A["V"]), 1.0, 0.0,
                        _d(lam), _d(lamB), _d(np.zeros(6 * n)), 0, corr, ex)


@pytest.mark.parametrize("combo", ["one-zero", "rho-SpSu"])
def test_mules_bodies(hk, orc, rbox, combo):  # noqa: F811
    b = rbox
    d = pc.mules_case(b, 4, combo)
    kw, n, nF, nB, L, U = d["kw"], d["n"], d["nF"], d["nB"], b.lower, b.upper
    H = Host(orc.Addr(n, L, U), dict(bfc=d["bfc"], diag=np.zeros(n), upper=np.zeros(nF), lower=None))
    bd, bdB = mo.upwind_flux(L, U, d["phi"], d["phiB"], d["psi"], d["psiB"])
    corr, corrB = d["phiPsi"] - bd, d["phiPsiB"] - bdB
    f = lambda x: None if x is None else np.ascontiguousarray(x, np.float64)
    A = {k: f(v) for k, v in dict(psi=d["psi"], psi0=d["psi0"], psiB=d["psiB"], bd=bd, bdB=bdB, corr=corr, corrB=corrB, V=d["V"],
                                  rho=kw.get("rho"), rho0=kw.get("rho0"), Sp=kw.get("Sp"), Su=kw.get("Su")).items()}
    for nIter in (0, 1, 3):
        lam, lamB = np.ones(nF), np.ones(nB)
        _limiter_call(hk, H, nIter, d["rDeltaT"], A, lam, lamB, n, 0, 0.0)
        want, wantB = mo.limiter(n, L, U, d["bfc"], d["V"], d["rDeltaT"], d["psi"], d["psi0"], d["psiB"], bd, bdB, corr, corrB, 1.0, 0.0,
                                 nIter, **kw)
        assert np.array_equal(lam, want) and np.array_equal(lamB, wantB), nIter
        assert nIter == 0 or (want < 1).sum() > nF // 10
    Ac = dict(A, psi0=A["psi"], corrB=f(corrB + 1e-5 * np.sin(np.arange(nB))))
    Ac.pop("bd"), Ac.pop("rho0")
    for ex in (0.0, 0.2):
        lam, lamB = np.ones(nF), np.ones(nB)
        Ac["bdB"] = f(d["phiB"])
        _limiter_call(hk, H, 3, d["rDeltaT"], Ac, lam, lamB, n, 1, ex)
        want, wantB = mo.limiter(n, L, U, d["bfc"], d["V"], d["rDeltaT"], d["psi"], d["psi"], d["psiB"], np.zeros(nF), d["phiB"], corr,
                                 Ac["corrB"], 1.0, 0.0, 3, kw.get("rho"), None, kw.get("Sp"), kw.get("Su"), corr=True, extremaCoeff=ex)
        assert np.array_equal(lam, want) and np.array_equal(lamB, wantB), ex


def test_limited_flux_and_interface_flux_bodies(hkv, orc, rbox):  # noqa: F811
    b = rbox
    d = _fields(b, 21)
    d["C"], d["cd"] = b.cell_centres(), b.weights()
    l, u = np.ascontiguousarray(b.lower, np.int32), np.ascontiguousarray(b.upper, np.int32)
    for scheme in sorted(lo.SCHEMES):
        for k in ((1.0, 0.5) if scheme == "limitedLinear" else (1.0,)):
            for fs in (1, -1):
                for os_ in (1, -1):
                    out = np.zeros(b.nFaces)
                    hkv.hk_limited_flux(b.nFaces, lo.SCHEMES[scheme], 2.0 / max(k, lo.SMALL), _d(l), _d(u), _d(d["flux"]), _d(d["vf"]),
                                        _d(d["g"]), _d(np.ascontiguousarray(d["C"])), _d(d["cd"]), fs, os_, _d(out))
                    want = io.limited_flux(scheme, l, u, d["flux"], d["vf"], d["g"], d["C"], d["cd"], k, fs, os_)
                    assert np.array_equal(out, want), (scheme, k, fs, os_)
    bfc = b.bFaceCells
    nB = len(bfc)
    H = Host(orc.Addr(b.nCells, b.lower, b.upper), dict(bfc=bfc, diag=np.zeros(b.nCells), upper=np.zeros(b.nFaces), lower=None))
    bSf = np.ascontiguousarray(b.bSf)
    bSn = np.random.default_rng(24).uniform(-1, 1, nB)
    bSn[::3] = 0.0
    Sf = np.ascontiguousarray(b.Sf())
    for deltaN in (1e-8, 0.5):
        for withPhi in (False, True):
            nHatf, nHatfB, phir = np.zeros(b.nFaces), np.zeros(nB), np.full(b.nFaces, -7.0)
            hkv.hk_interface_flux(H.p(), _d(d["w"]), _d(d["g"]), _d(Sf), _d(bSf), _d(bSn), deltaN, _d(d["flux"]) if withPhi else None,
                                  _d(d["magSf"]), 0.75, _d(nHatf), _d(nHatfB), _d(phir))
            w0, w1, w2 = io.interface_flux(b.lower, b.upper, d["w"], d["g"], Sf, bfc, bSf, bSn, deltaN, d["flux"] if withPhi else None,
                                           d["magSf"], 0.75)
            assert np.array_equal(nHatf, w0) and np.array_equal(nHatfB, w1), (deltaN, withPhi)
            assert np.array_equal(phir, w2) if withPhi else (phir == -7.0).all()


# ---- independent references on the oracle's outputs ----------------------------------------------------------------------
def test_gauss_grad_and_closed_sum_bounds_hold_for_the_oracle(orc):
    b = pc.refined_box(5, "random", seed=8)
    a = pc.addr(orc, b)
    a_, b_ = np.array([0.7, -1.3, 2.1]), 0.4
    phif, phib = b.face_centres() @ a_ + b_, b.bCf @ a_ + b_
    got = np.asarray(orc.gauss_grad(a, b.Sf().ravel(), phif, b.bFaceCells, b.bSf.ravel(), phib, b.volumes(), 1)).reshape(-1, 3)
    pc.check_exact_gauss_grad(b, phif, phib, got, a_)
    with pytest.raises(AssertionError):           # a face counted twice leaves the bound
        pc.check_exact_gauss_grad(b, phif, phib, got + np.where(np.arange(b.nCells) == 17, 1e-9, 0.0)[:, None], a_)
    U = np.array([0.3, -0.8, 1.1])
    got = np.asarray(orc.surface_integrate(a, b.Sf() @ U, b.bFaceCells, b.bSf @ U, b.volumes(), 1, False, -1))
    pc.check_closed_sum(b, U, got)


def test_matrix_product_bounds_hold_for_the_oracle(orc):
    from test_gpu_engine_streams import Mismatches
    b = pc.refined_box(6, "random", seed=5)
    a, diag, up, low = pc.asym_matrix(orc, b)
    om = orc.Matrix(a, diag, up, low)
    rng = np.random.default_rng(3)
    x, rhs = rng.uniform(-1, 1, b.nCells), rng.uniform(-1, 1, b.nCells)
    M = Mismatches()
    got = dict(Amul=om.amul(x), Tmul=om.tmul(x), residual=om.residual(x, rhs))
    pc.check_matrix_products(M, b.lower, b.upper, diag, up, low, x, rhs, got)
    M.check()
    M = Mismatches()
    pc.check_matrix_products(M, b.lower, b.upper, diag, up, low, x, rhs, dict(got, Tmul=om.amul(x)))   # a wrong transpose is seen
    assert len(M.msgs) == 1


def test_interface_normal_bound_holds_for_the_oracle():
    b = pc.refined_box(4, "coarse-first")
    a_ = np.array([0.3, -0.5, 0.8])
    bSn = np.zeros(len(b.bFaceCells))
    w0, _, _ = io.interface_flux(b.lower, b.upper, b.weights(), np.tile(a_, (b.nCells, 1)), b.Sf(), b.bFaceCells, b.bSf, bSn, 1e-8,
                                 None, b.magSf(), 0.75)
    pc.check_interface_normal(b, a_, 1e-8, w0)


def test_mules_rotation_is_bounded_and_conservative_with_the_oracle(orc):
    b = pc.refined_box(8, "random", seed=3)
    a = pc.addr(orc, b)
    V, bfc = b.volumes(), b.bFaceCells

    def step(psi, phi, phiB, psiB, dt, limited):
        phiPsi = phi * np.asarray(orc.interpolate_linear(a, b.weights(), psi, 1))
        phiPsiB = phiB * psiB
        if limited:
            phiPsi, phiPsiB = mo.limit(b.nCells, b.lower, b.upper, bfc, V, 1 / dt, psi, psi, psiB, phi, phiB, phiPsi, phiPsiB, 1.0, 0.0, 3)
        return mo.explicit_solve(b.nCells, b.lower, b.upper, bfc, V, 1 / dt, psi, phiPsi, phiPsiB), phiPsiB
    pc.check_mules_rotation(b, step)


def test_dense_reference_of_the_fvm_cases(orc):
    """the cases of test_gpu_polymesh.test_fvm_solve are non-singular and the oracle's solve reaches the dense solution"""
    from test_oracle_fvm import make
    b = pc.refined_box(4, "random", seed=2)
    for nc, solver, pre in ((1, "PCG", "DIC"), (3, "PBiCG", "DILU")):
        a, d, _ = pc.fvm_case(orc, b, nc, 4)
        psi, perfs, _ = make(orc, a, d, nc).solve(solver, pre, tolerance=1e-12, maxIter=1000)
        for k in range(nc):
            Ad, rhs = full_system(b, d, k)
            np.testing.assert_allclose(psi[:, k], np.linalg.solve(Ad, rhs), rtol=0, atol=1e-9)


# ---- dry run of the GPU module -------------------------------------------------------------------------------------------
def test_gpu_module_over_the_oracle_stand_in(monkeypatch, orc):
    """tests/test_gpu_polymesh.py's own logic (indexing, shapes, tolerances) over tests/oracle_backend.py, wherever the stand-in has
    the entry point; the engine-, band- and stream-specific parts skip themselves"""
    import oracle_backend
    import test_gpu_polymesh as G
    monkeypatch.setenv("B200LDU_DRYRUN_ORACLE", "1")
    gpu = oracle_backend.fixture()
    for kind in G.KINDS + ["periodic"]:
        G.test_face_sums(gpu, orc, kind)
    G.test_gauss_grad_of_a_linear_field_is_exact(gpu, orc)
    for kind in ("random", "periodic"):
        for nc in (1, 3):
            G.test_fvm_operations(gpu, orc, kind, nc)
    for nc, solver, pre in ((1, "PCG", "DIC"), (3, "PBiCG", "DILU"), (1, "GAMG", "GaussSeidel")):
        G.test_fvm_solve(gpu, orc, "periodic" if solver != "GAMG" else "random", nc, solver, pre)
    for kind in ("fine-first", "graph"):
        G.test_mules(gpu, kind, "rho-SpSu")
    G.test_mules_step_is_bounded_and_conservative(gpu)
