"""b200ldu_launch_count is the number of library kernels launched: for every non-solver entry point that launches
kernels, the change of the counter over one call equals the number of kernels the CUDA profiler records for it
(memset and memcpy activities are not kernels).  Meshes: a hex box with a boundary-face list and a cyclic patch pair,
and a one-cell addressing without faces; matrices with absent arrays; one and three components."""
import ctypes as C
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def hex_cyclic_case(meshmod):
    """6x5x4 hex box, periodic in x: the x-min and x-max faces are a cyclic pair, the other walls the boundary list"""
    nx, ny, nz = 6, 5, 4
    m = meshmod.hex_mesh(nx, ny, nz)
    jk = np.arange(ny * nz)
    lo, hi = (jk * nx).astype(np.int32), (jk * nx + nx - 1).astype(np.int32)
    patches = dict(patchStart=np.array([0, ny * nz, 2 * ny * nz], np.int32), faceCells=np.concatenate([lo, hi]),
                   neighbRank=np.array([-2, -1], np.int32), cellCentres=m.cell_centres())
    walls = np.concatenate([p.faceCells for p in m.wall_patches() if p.name not in ("xmin", "xmax")]).astype(np.int32)
    return m.nCells, m.lower, m.upper, patches, walls


def one_cell_case():
    return 1, np.zeros(0, np.int32), np.zeros(0, np.int32), {}, np.zeros(0, np.int32)


def entry_point_calls(capi, ctx, torch, case, nc):
    """(name, call) of every entry point under test on one addressing; every tensor is allocated here, before any
    call, so that the calls themselves launch nothing but the library's kernels"""
    L = capi.lib()
    nCells, lower, upper, patches, bfc = case
    nF, nB = len(lower), len(bfc)
    nPF = int(patches["patchStart"][-1]) if patches else 0
    addr = capi.LduAddressing(ctx, nCells, lower, upper, **patches)
    plain = capi.LduAddressing(ctx, nCells, lower, upper)  # the same mesh without coupled patches
    capi.fv_boundary_set(addr, bfc)
    rng = np.random.default_rng(3)
    dev = ctx.device

    def f(n, lo=0.5, hi=1.5):
        return torch.from_numpy(rng.uniform(lo, hi, max(n, 1))).to(dev)

    def p(t):
        return capi._dp(t)

    V, w, dc = f(nCells), f(nF, 0.2, 0.8), f(nF)
    diag, up, lw, bou, inc = f(nCells, 4, 5), f(nF, -1, -0.5), f(nF, -1, -0.5), f(nPF), f(nPF)
    psi, src, vf, pnf = f(nCells * nc, -1, 1), f(nCells * nc), f(nCells * nc, -1, 1), f(nPF * nc)
    ic, bc = f(nB * nc), f(nB * nc)
    Sf, bSf, bvf, ssf, bssf = f(nF * 3), f(nB * 3), f(nB * nc), f(nF * nc, -1, 1), f(nB * nc)
    U, C3, gradc, phi = f(nCells * 3, -1, 1), f(nCells * 3), f(nCells * 3, -1, 1), f(nF, -1, 1)
    out = [f(max(nCells, nF, nB, nPF) * 9) for _ in range(4)]
    o = [p(t) for t in out]
    cells = torch.from_numpy(rng.integers(0, nCells, 7).astype(np.int32)).to(dev)
    T9 = f(nCells * 9, -1, 1)
    one = torch.ones(max(nF, 1), dtype=torch.float64, device=dev)
    lam, lamB = one.clone(), torch.ones(max(nB + nPF, 1), dtype=torch.float64, device=dev)
    psiB, phiB, phiCorrB = f(nB + nPF, -1, 1), f(nB + nPF, -1, 1), f(nB + nPF, -1, 1)
    mat = capi.LduMatrix(addr)
    mat0 = capi.LduMatrix(plain)
    A = dict(d=f(nCells), u=f(nF), l=f(nF))
    B = dict(d=f(nCells), u=f(nF), l=f(nF))
    iface = (p(bou), p(inc)) if nPF else (None, None)
    ref = np.array([0.5, -1.25, 2.0][:nc])

    def has(*flags):
        return (C.c_int * 3)(*flags)

    def mules_boundary():  # MULES wants the coupled faces last in the boundary list
        capi.fv_boundary_set(addr, np.concatenate([bfc, patches["faceCells"]]) if nPF else bfc)

    calls = [
        ("matrix_set symmetric, no interfaces", lambda: L.b200ldu_matrix_set(mat0.h, p(diag), p(up), None, None, None)),
        ("matrix_set asymmetric, no interfaces", lambda: L.b200ldu_matrix_set(mat0.h, p(diag), p(up), p(lw), None, None)),
        ("matrix_set symmetric, one interface array", lambda: L.b200ldu_matrix_set(mat.h, p(diag), p(up), None, iface[0], iface[0])),
        ("matrix_set symmetric", lambda: L.b200ldu_matrix_set(mat.h, p(diag), p(up), None, *iface)),
        ("matrix_set asymmetric", lambda: L.b200ldu_matrix_set(mat.h, p(diag), p(up), p(lw), *iface)),
        ("to_banded", lambda: L.b200ldu_to_banded(addr.h, p(V), o[0])),
        ("from_banded", lambda: L.b200ldu_from_banded(addr.h, o[0], o[1])),
        ("amul", lambda: L.b200ldu_amul(mat.h, p(V), o[0])),
        ("tmul", lambda: L.b200ldu_tmul(mat.h, p(V), o[0])),
        ("sumA", lambda: L.b200ldu_sumA(mat.h, o[0])),
        ("residual", lambda: L.b200ldu_residual(mat.h, p(V), p(diag), o[0])),
        ("H", lambda: L.b200ldu_H(mat.h, p(V), o[0])),
        ("H1", lambda: L.b200ldu_H1(mat.h, o[0])),
        ("fv_surface_integrate", lambda: L.b200ldu_fv_surface_integrate(addr.h, nc, p(ssf), p(bssf), p(V), o[0], 1, -1)),
        ("fv_gauss_grad", lambda: L.b200ldu_fv_gauss_grad(addr.h, nc, p(Sf), p(ssf), p(bSf), p(bssf), p(V), o[0])),
        ("fv_laplacian_fill", lambda: L.b200ldu_fv_laplacian_fill(addr.h, p(dc), p(w), o[0], o[1])),
        ("fv_convection_fill", lambda: L.b200ldu_fv_convection_fill(addr.h, p(w), p(phi), o[0], o[1], o[2])),
        ("fv_interpolate_linear", lambda: L.b200ldu_fv_interpolate_linear(addr.h, nc, p(w), p(vf), o[0])),
        ("fv_grad_linear", lambda: L.b200ldu_fv_grad_linear(addr.h, nc, p(Sf), p(w), p(vf), p(bSf), p(bvf), p(V), o[0])),
        ("fv_flux_linear", lambda: L.b200ldu_fv_flux_linear(addr.h, p(Sf), p(w), p(U), o[0])),
        ("fv_add_boundary_diag", lambda: L.b200ldu_fv_add_boundary_diag(addr.h, p(ic), o[0])),
        ("fv_add_boundary_source", lambda: L.b200ldu_fv_add_boundary_source(addr.h, p(bc), o[0])),
        ("fv_patch_neighbour_field", lambda: L.b200ldu_fv_patch_neighbour_field(addr.h, nc, p(vf), o[0])),
        ("fv_sngrad", lambda: L.b200ldu_fv_sngrad(addr.h, nc, p(dc), p(vf), o[0])),
        ("fv_limiter upwind", lambda: L.b200ldu_fv_limiter(addr.h, b"upwind", 1.0, None, None, None, None, o[0])),
        ("fv_limiter limitedLinear",
         lambda: L.b200ldu_fv_limiter(addr.h, b"limitedLinear", 1.0, p(phi), p(vf), p(gradc), p(C3), o[0])),
        ("fv_limited_weights", lambda: L.b200ldu_fv_limited_weights(ctx.h, nF, p(w), p(w), p(phi), o[0])),
        ("fvm_add_boundary_diag", lambda: L.b200ldu_fvm_add_boundary_diag(mat.h, nc, nc - 1, p(ic), p(diag), o[0])),
        ("fvm_add_boundary_diag average", lambda: L.b200ldu_fvm_add_boundary_diag(mat.h, nc, -1, p(ic), p(diag), o[0])),
        ("fvm_add_boundary_source", lambda: L.b200ldu_fvm_add_boundary_source(mat.h, nc, p(bc), p(pnf), p(src), o[0])),
        ("fvm_A", lambda: L.b200ldu_fvm_A(mat.h, nc, p(ic), p(V), o[0])),
        ("fvm_H", lambda: L.b200ldu_fvm_H(mat.h, nc, p(psi), p(src), p(bc), p(pnf), p(V), o[0])),
        ("fvm_flux", lambda: L.b200ldu_fvm_flux(mat.h, nc, p(psi), p(ic), p(bc), p(pnf), o[0], o[1], o[2])),
        ("fvm_relax", lambda: L.b200ldu_fvm_relax(mat.h, nc, 0.7, p(psi), p(ic), o[0], o[1])),
        ("fvm_set_reference",
         lambda: L.b200ldu_fvm_set_reference(mat.h, 0, nc, ref.ctypes.data_as(C.c_void_p), o[0], o[1])),
        ("ldu_row_sum sumDiag", lambda: L.b200ldu_ldu_row_sum(addr.h, 0, p(up), None, o[0])),
        ("ldu_row_sum sumMagOffDiag", lambda: L.b200ldu_ldu_row_sum(addr.h, 2, p(up), p(lw), o[0])),
        ("ldu_add_assign symmetric += asymmetric", lambda: L.b200ldu_ldu_add_assign(
            addr.h, 0, p(A["d"]), p(A["u"]), p(A["l"]), has(1, 1, 0), p(B["d"]), p(B["u"]), p(B["l"]), has(1, 1, 1))),
        ("ldu_add_assign diagonal -= symmetric", lambda: L.b200ldu_ldu_add_assign(
            addr.h, 1, p(A["d"]), p(A["u"]), None, has(1, 0, 0), p(B["d"]), p(B["u"]), None, has(1, 1, 0))),
        ("ldu_add_assign += diagonal, absent triangles", lambda: L.b200ldu_ldu_add_assign(
            addr.h, 0, p(A["d"]), None, None, has(1, 0, 0), p(B["d"]), None, None, has(1, 0, 0))),
        ("ldu_scale asymmetric by a field", lambda: L.b200ldu_ldu_scale(addr.h, p(V), 0.0, p(A["d"]), p(A["u"]), p(A["l"]),
                                                                        has(1, 1, 1))),
        ("ldu_scale diagonal, absent triangles", lambda: L.b200ldu_ldu_scale(addr.h, None, 2.0, p(A["d"]), None, None,
                                                                             has(1, 0, 0))),
        ("ldu_scale symmetric, absent lower", lambda: L.b200ldu_ldu_scale(addr.h, None, 2.0, p(A["d"]), p(A["u"]), None,
                                                                          has(1, 1, 0))),
        ("field_binary", lambda: L.b200ldu_field_binary(ctx.h, 2, nCells, 1, p(V), nc, p(vf), o[0])),
        ("field_unary", lambda: L.b200ldu_field_unary(ctx.h, 1, nCells * nc, 0.0, p(vf), o[0])),
        ("field_dot3", lambda: L.b200ldu_field_dot3(ctx.h, nCells, p(U), p(C3), o[0])),
        ("field_symm_magsqr", lambda: L.b200ldu_field_symm_magsqr(ctx.h, nCells, p(T9), o[0])),
        ("field_gather", lambda: L.b200ldu_field_gather(ctx.h, cells.numel(), nc, p(cells), p(vf), o[0])),
        ("fv_boundary_set with the coupled faces last", mules_boundary),
        ("mules_limiter", lambda: L.b200ldu_mules_limiter(
            addr.h, 2, 10.0, None, None, p(V), p(V), p(psiB), p(phi), p(phiB), p(phi), p(phiCorrB), None, None, p(V),
            1.5, 0.5, p(lam), p(lamB), nPF)),
        ("mules_limiter_corr", lambda: L.b200ldu_mules_limiter_corr(
            addr.h, 2, 10.0, None, p(V), p(psiB), p(phiB), p(phi), p(phiCorrB), None, None, p(V), 1.5, 0.5, 0.1, p(lam),
            p(lamB), nPF)),
    ]
    if nF:
        calls.insert(13, ("faceH", lambda: L.b200ldu_faceH(mat.h, p(V), o[0])))
    if nc == 1:
        calls.insert(-3, ("fvm_residual", lambda: L.b200ldu_fvm_residual(mat.h, p(psi), p(src), p(ic), p(bc), p(pnf), o[0])))
    keep = (addr, plain, mat, mat0, out)
    return calls, keep


def device_kernels(torch, fn):
    """(return value of fn, number of kernels the profiler records while it runs)"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rc = fn()
        torch.cuda.synchronize()
    n = sum(1 for e in prof.profiler.kineto_results.events()
            if e.device_type() == DeviceType.CUDA and not e.name().startswith(("Memcpy", "Memset")))
    return rc, n


@pytest.mark.parametrize("mesh", ["hex_cyclic", "one_cell"])
@pytest.mark.parametrize("nc", [1, 3])
def test_launch_count_matches_the_profiler(meshmod, mesh, nc):
    import torch
    assert torch.cuda.is_available()
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    case = hex_cyclic_case(meshmod) if mesh == "hex_cyclic" else one_cell_case()
    calls, keep = entry_point_calls(capi, ctx, torch, case, nc)
    device_kernels(torch, lambda: None)  # profiler start-up outside the measured calls
    wrong = []
    for name, call in calls:
        before = ctx.launches
        rc, kernels = device_kernels(torch, call)
        if rc:
            wrong.append(f"{name}: error {rc}, {capi.lib().b200ldu_last_error().decode(errors='replace')}")
        elif ctx.launches - before != kernels:
            wrong.append(f"{name}: counted {ctx.launches - before}, profiler {kernels}")
    assert not wrong, "\n".join(wrong)
    for h in keep[:4][::-1]:
        h.close()
    ctx.close()
