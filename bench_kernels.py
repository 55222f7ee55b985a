#!/usr/bin/env python
"""Per-kernel roofline table (not the driver's bench contract -- that is bench.py):
times every hot-path kernel alone on the 256^3 cavity with CUDA events and reports achieved
ALGORITHMIC GB/s (SURVEY.md section 8d byte counts) against the measured HBM peak.
  python bench_kernels.py [--n 256] [--reps 20] > gpurun_out/kernels.json
The two sweeps of the fused PCG iteration are timed inside a 50-iteration solve with torch.profiler, in a process of
its own (`--pcg-sweeps` runs only that part): per-sweep time, layout bytes and GB/s, and the gaps between the sweeps.
Run it under `ncu --metrics gpu__time_duration.sum` for the matching launch list."""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def pcg_sweep_bytes(info):
    """Bytes the banded layout moves in the two sweeps of one fused PCG iteration (single domain: every entry is
    local).  Stream: the face stream's stored owner slots and list items, an 8 B coefficient each, plus its table of
    4 B column and product-slot words once, or, for a layout without one, the entry stream's 8 B coefficient + 2 B
    column per entry.  Halo: a 4 B haloIdx per column plus the vectors the op's stage() reads there.  Own rows: the
    vectors read and written while staging and in finish()."""
    nPad, nE, nH = info["nPadRows"], info["nEntries"], info["nHalo"]
    if info.get("faceStream"):
        stream = 8 * (info["fsOwnerSlots"] + info["fsListItems"]) + 4 * info["fsTemplateWords"]
    else:
        stream = 10 * nE
    # A (PcgAinvOp): own rows read rOld, w, rD and write rNew, z; halo reads w, rOld, rD
    a = 40 * nPad + stream + (4 + 24) * nH
    # B (PcgAmulOp): own rows read z, pOld, psi, diag and write pNew, psi, w; halo reads z, pOld
    b = 56 * nPad + stream + (4 + 16) * nH
    return a, b


def pcg_sweeps(n, iters):
    """Per-kernel times of the two fused PCG sweeps inside an n^3, `iters`-iteration PCG+DIC solve, from
    torch.profiler (CUDA activities), and the gaps between consecutive sweeps.  Prints one JSON object."""
    import tempfile

    import torch
    from torch.profiler import ProfilerActivity, profile
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    meshmod = importlib.import_module("rapidcfd-dev_b200.mesh")
    mesh = meshmod.hex_mesh(n)
    ctx = capi.Context(0)
    dev = ctx.device
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    addr = capi.mesh_to_device(ctx, mesh)
    cp = meshmod.pressure_laplacian(mesh)
    mat = capi.LduMatrix(addr)
    mat.set(tt(cp["diag"]), tt(cp["upper"]))
    b = tt(meshmod.cell_field_global(mesh, 9))
    psi = torch.zeros(mesh.nCells, dtype=torch.float64, device=dev)
    kw = dict(tolerance=0.0, maxIter=iters - 1)
    for _ in range(2):
        psi.zero_()
        mat.solve("PCG", "DIC", psi, b, **kw)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            psi.zero_()
            mat.solve("PCG", "DIC", psi, b, **kw)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    kern = sorted((e for e in trace.get("traceEvents", []) if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    # the solve's close (pcg_close_kernel: last alpha, r and sum|r| without the preconditioner) is neither sweep
    which = lambda e: "A" if "PcgAinvOp" in e["name"] else ("B" if "PcgAmulOp" in e["name"] else None)
    dur = {"A": [], "B": []}
    gap = {"A->B": [], "B->A": []}
    prev = None
    for e in kern:
        w = which(e)
        if w is None:
            prev = None
            continue
        dur[w].append(e["dur"])
        if prev is not None and which(prev) != w:
            gap[f"{which(prev)}->{w}"].append(e["ts"] - (prev["ts"] + prev["dur"]))
        prev = e
    info = addr.info()
    bytesA, bytesB = pcg_sweep_bytes(info)
    med = lambda v: float(np.median(v)) if v else float("nan")
    rows = []
    for w, nm, nb in (("A", "PCG sweep A (AINV + r update)", bytesA), ("B", "PCG sweep B (psi/p update + Amul)", bytesB)):
        us = med(dur[w])
        rows.append({"kernel": nm, "layout_bytes": int(nb), "us_median": us, "us_min": min(dur[w], default=float("nan")),
                     "launches": len(dur[w]), "GBps": nb / (us * 1e-6) / 1e9})
    out = {"n": n, "iters": iters, "layout": info, "sweeps": rows,
           "gap_us_median": {k: med(v) for k, v in gap.items()}, "gaps": {k: len(v) for k, v in gap.items()},
           "iteration_us": med(dur["A"]) + med(dur["B"]) + med(gap["A->B"]) + med(gap["B->A"]),
           "close_us_median": med([e["dur"] for e in kern if "pcg_close_kernel" in e["name"]])}
    mat.close()
    addr.close()
    ctx.close()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--pcg-sweeps", action="store_true",
                    help="only the per-sweep attribution of the fused PCG iteration (torch.profiler)")
    args = ap.parse_args()
    if args.pcg_sweeps:
        return pcg_sweeps(args.n, 50)
    import subprocess
    # the profiler runs in a process of its own: tracing must not slow down the event-timed rows below
    sw = subprocess.run([sys.executable, os.path.abspath(__file__), "--pcg-sweeps", "--n", str(args.n)],
                        capture_output=True, text=True)
    sweeps = json.loads(sw.stdout.strip().splitlines()[-1]) if sw.returncode == 0 else {"error": sw.stderr[-2000:]}
    for r in sweeps.get("sweeps", []):
        print(f"{r['kernel']:34s} {r['us_median']:9.1f} us  {r['GBps']:8.1f} GB/s (layout bytes)", file=sys.stderr)
    print("gaps between sweeps (us):", sweeps.get("gap_us_median"), file=sys.stderr)
    import torch
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    meshmod = importlib.import_module("rapidcfd-dev_b200.mesh")
    from bench import peaks
    peak, peak_src = peaks()
    L = capi.lib()
    n = args.n
    mesh = meshmod.hex_mesh(n)
    N, F = mesh.nCells, mesh.nFaces
    ctx = capi.Context(0)
    dev = ctx.device
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    addr = capi.mesh_to_device(ctx, mesh)
    dp = capi._dp
    rows = []

    def timeit(name, nbytes, fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        gbs = nbytes / (ms * 1e-3) / 1e9
        rows.append({"kernel": name, "algorithmic_bytes": int(nbytes), "ms": ms, "GBps": gbs, "frac": gbs / peak})
        print(f"{name:34s} {ms*1e3:9.1f} us  {gbs:8.1f} GB/s  {gbs/peak:5.2f}", file=sys.stderr)

    vl = addr.vec_len
    xb = torch.rand(vl, dtype=torch.float64, device=dev)
    yb = torch.zeros(vl, dtype=torch.float64, device=dev)
    bb = torch.rand(vl, dtype=torch.float64, device=dev)
    xb[N:] = 0
    # ---- symmetric matrix ----
    cp = meshmod.pressure_laplacian(mesh)
    mat = capi.LduMatrix(addr)
    dg, up = tt(cp["diag"]), tt(cp["upper"])
    mat.set(dg, up)
    op = lambda nm: (lambda: capi.check(L.b200ldu_bench_op(mat.h, nm.encode(), dp(xb), dp(yb), dp(bb))))
    timeit("Amul symmetric", 24 * N + 16 * F, op("amul"))
    timeit("Amul + fused <Ap,p>", 24 * N + 16 * F, op("amul_dot"))
    timeit("AINV precondition", 24 * N + 16 * F, op("ainv"))
    timeit("AINV + fused <w,r>", 24 * N + 16 * F, op("ainv_dot"))
    timeit("Jacobi sweep", 40 * N + 16 * F, op("jacobi"))
    timeit("residual + fused sum|r|", 32 * N + 16 * F, op("residual"))
    timeit("sumA", 16 * N + 8 * F, op("sumA"))
    mat.close()
    # ---- asymmetric matrix ----
    cu = meshmod.momentum_matrix(mesh)
    matU = capi.LduMatrix(addr)
    dgu, upu, lou = tt(cu["diag"]), tt(cu["upper"]), tt(cu["lower"])
    matU.set(dgu, upu, lou)
    opu = lambda nm: (lambda: capi.check(L.b200ldu_bench_op(matU.h, nm.encode(), dp(xb), dp(yb), dp(bb))))
    timeit("Amul asymmetric", 24 * N + 24 * F, opu("amul"))
    timeit("Tmul asymmetric", 24 * N + 24 * F, opu("tmul"))
    psi, src = torch.rand(N, dtype=torch.float64, device=dev), torch.rand(N, dtype=torch.float64, device=dev)
    timeit("faceH (flux)", 24 * F + 8 * N, lambda: matU.faceH(psi))
    matU.close()
    del dgu, upu, lou
    # ---- vector kernels through a short PCG (fused op list): whole-iteration rate ----
    # ---- finite-volume face sums ----
    bfc = np.concatenate([p.faceCells for p in mesh.patches]).astype(np.int32)
    capi.check(L.b200ldu_fv_boundary_set(addr.h, len(bfc), bfc.ctypes.data))
    nB = len(bfc)
    V = tt(mesh.volumes())
    for nc in (1, 3):
        ssf = torch.rand(F * nc, dtype=torch.float64, device=dev)
        bssf = torch.rand(nB * nc, dtype=torch.float64, device=dev)
        out = torch.empty(N * nc, dtype=torch.float64, device=dev)
        timeit(f"fvc::surfaceIntegrate nComp={nc}", 8 * nc * F + 8 * F + 8 * N + 8 * nc * N,
               lambda: capi.check(L.b200ldu_fv_surface_integrate(addr.h, nc, dp(ssf), dp(bssf), dp(V), dp(out), 1, -1)))
        Sf = torch.rand(F * 3, dtype=torch.float64, device=dev)
        bSf = torch.rand(nB * 3, dtype=torch.float64, device=dev)
        g = torch.empty(N * 3 * nc, dtype=torch.float64, device=dev)
        timeit(f"gaussGrad::gradf nComp={nc}", 8 * nc * F + 24 * F + 8 * F + 8 * N + 24 * nc * N,
               lambda: capi.check(L.b200ldu_fv_gauss_grad(addr.h, nc, dp(Sf), dp(ssf), dp(bSf), dp(bssf), dp(V), dp(g))))
        vf = torch.rand(N * nc, dtype=torch.float64, device=dev)
        w = torch.rand(F, dtype=torch.float64, device=dev)
        sf = torch.empty(F * nc, dtype=torch.float64, device=dev)
        timeit(f"linear interpolate nComp={nc}", 8 * F + 8 * F + 8 * nc * N + 8 * nc * F,
               lambda: capi.check(L.b200ldu_fv_interpolate_linear(addr.h, nc, dp(w), dp(vf), dp(sf))))
        # fused: grad(interpolate(vf)) without the F-sized face field (algorithmic bytes of the
        # fused op: Sf + w + addressing once, vf read, grad written)
        bvf = torch.rand(nB * nc, dtype=torch.float64, device=dev)
        timeit(f"fused linear-interpolate + gaussGrad nComp={nc}", 24 * F + 8 * F + 8 * F + 8 * nc * N + 8 * N + 24 * nc * N,
               lambda: capi.check(L.b200ldu_fv_grad_linear(addr.h, nc, dp(Sf), dp(w), dp(vf), dp(bSf), dp(bvf), dp(V), dp(g))))
        if nc == 3:
            phi = torch.empty(F, dtype=torch.float64, device=dev)
            timeit("fused flux phi = interpolate(U) & Sf", 24 * F + 8 * F + 8 * F + 24 * N + 8 * F,
                   lambda: capi.check(L.b200ldu_fv_flux_linear(addr.h, dp(Sf), dp(w), dp(vf), dp(phi))))
            del phi
        del ssf, bssf, out, Sf, bSf, g, vf, w, sf, bvf
    dc, gm = torch.rand(F, dtype=torch.float64, device=dev), torch.rand(F, dtype=torch.float64, device=dev)
    upp, low = torch.empty(F, dtype=torch.float64, device=dev), torch.empty(F, dtype=torch.float64, device=dev)
    dgo = torch.empty(N, dtype=torch.float64, device=dev)
    timeit("fvm::laplacian fill (+negSumDiag)", 24 * F + 8 * F + 8 * N,
           lambda: capi.check(L.b200ldu_fv_laplacian_fill(addr.h, dp(dc), dp(gm), dp(upp), dp(dgo))))
    timeit("fvm::div fill (+negSumDiag)", 32 * F + 8 * F + 8 * N,
           lambda: capi.check(L.b200ldu_fv_convection_fill(addr.h, dp(dc), dp(gm), dp(low), dp(upp), dp(dgo))))
    # ---- explicit MULES: limiter (3 sweeps) and the whole limit + explicitSolve update ----
    try:
        mules = importlib.import_module("rapidcfd-dev_b200.mules")
        ps_, bfc_ = mesh.patch_start_facecells(mesh.wall_patches())
        capi.fv_boundary_set(addr, bfc_)
        nBm = len(bfc_)
        ops = capi.FieldOps(ctx)
        Vm = tt(mesh.volumes())
        psi_m = torch.rand(N, dtype=torch.float64, device=dev)
        phi_m = (torch.rand(F, dtype=torch.float64, device=dev) - 0.5) * (mesh.h ** 2)
        zB = torch.zeros(nBm, dtype=torch.float64, device=dev)
        wl = torch.full((F,), 0.5, dtype=torch.float64, device=dev)
        phiPsi = ops.mul(phi_m, capi.fv_interpolate_linear(addr, 1, wl, psi_m))
        bd, bdB = mules.upwind_flux(capi, addr, ops, phi_m, zB, psi_m, zB)
        corr = ops.sub(phiPsi, bd)
        rdt = 4.0 / mesh.h
        # bounds kernel: psi, psi0, V, 4 outputs (56N) + phiBD, phiCorr (16F); per sweep: lambda, phiCorr (16F) + 4 budgets in,
        # 2 cell limiters out (48N), then phiCorr, lambda in, lambda out (24F) + the cell limiters gathered (counted once, 16N)
        timeit("MULES::limiter, 3 sweeps (7 launches)", 56 * N + 16 * F + 3 * (64 * N + 40 * F),
               lambda: capi.mules_limiter(addr, Vm, rdt, psi_m, psi_m, zB, bd, zB, corr, zB, 1.0, 0.0, 3))
        timeit("MULES::limit + explicitSolve (ABI compositions)", 56 * N + 16 * F + 3 * (64 * N + 40 * F) + 80 * F + 56 * N,
               lambda: mules.explicit_solve(capi, addr, ops, Vm, rdt, psi_m,
                                            *mules.limit(capi, addr, ops, Vm, rdt, psi_m, psi_m, zB, phi_m, zB, phiPsi, zB, 1.0, 0.0, 3)))
        del Vm, psi_m, phi_m, zB, wl, phiPsi, bd, bdB, corr
    except Exception as e:  # noqa: BLE001 -- keep the table above
        print("MULES rows:", repr(e), file=sys.stderr)
    # ---- time to solution: GAMG vs PCG on the pressure matrix (tolerance 1e-6, relTol 0) ----
    import time
    del dc, gm, upp, low, dgo
    solves = {}
    mat = capi.LduMatrix(addr)
    mat.set(dg, up)
    b = tt(meshmod.cell_field_global(mesh, 9))
    t0 = time.perf_counter()
    gg = capi.GamgAgglomeration(addr, meshmod.face_area_pair_weights(mesh), 10)
    t_agg = time.perf_counter() - t0
    for name, solver, second, kw in (("GAMG", "GAMG", "GaussSeidel", dict(tolerance=1e-6, maxIter=200)),
                                     ("PCG+DIC", "PCG", "DIC", dict(tolerance=1e-6, maxIter=5000))):
        for rep in range(2):
            psi = torch.zeros(N, dtype=torch.float64, device=dev)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            perf, _ = mat.solve(solver, second, psi, b, gamg=gg if solver == "GAMG" else None, **kw)
            e1.record()
            torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        solves[name] = {"ms": ms, "iterations": perf.nIterations, "final_residual": perf.finalResidual,
                        "Mcell_iters_per_s": N * perf.nIterations / (ms * 1e-3) / 1e6, "line": perf.line("p")}
        print(name, solves[name], file=sys.stderr)
    solves["GAMG"]["levels"] = gg.nLevels
    solves["GAMG"]["agglomeration_host_s"] = t_agg
    # ---- fvMatrix glue (row a17, csrc/fvmatrix.cu): last, and guarded -- first GPU run is still to come ----
    fvm_error = None
    try:
        for nc in (1, 3):
            psi = torch.rand(N * nc, dtype=torch.float64, device=dev)
            src = torch.rand(N * nc, dtype=torch.float64, device=dev)
            ic = torch.rand(nB * nc, dtype=torch.float64, device=dev)
            bcf = torch.rand(nB * nc, dtype=torch.float64, device=dev)
            dgc = dg.clone()
            fv = capi.FvMatrix(mat, nc, dgc, src, psi, V, ic, bcf)
            timeit(f"fvMatrix::A nComp={nc}", 24 * N, fv.A)
            timeit(f"fvMatrix::H nComp={nc}", 16 * F + 8 * F + (16 * nc + 8) * N + 8 * nc * N, fv.H)
            timeit(f"fvMatrix::flux nComp={nc}", 16 * F + 8 * F + 8 * nc * N + 8 * nc * F, lambda: fv.flux(nB))
            timeit(f"fvMatrix::relax nComp={nc}", 16 * F + 16 * N + 24 * nc * N, lambda: fv.relax(0.9))
            tmpd = dg.clone()
            timeit(f"fvMatrix::addBoundaryDiag nComp={nc}", 16 * N, lambda: fv.addBoundaryDiag(tmpd, 0))
            timeit(f"fvMatrix::addBoundarySource nComp={nc}", 16 * nc * N, lambda: fv.addBoundarySource(src))
            if nc == 1:
                timeit("fvMatrix::residual", 16 * F + 8 * F + 40 * N, fv.residual)
            del psi, src, ic, bcf, dgc, tmpd
        # solveSegregated overhead: fold + two coefficient re-streams around a fixed 20-iteration PCG
        psi = torch.zeros(N, dtype=torch.float64, device=dev)
        ic = torch.rand(nB, dtype=torch.float64, device=dev) * -1e-3
        bcf = torch.rand(nB, dtype=torch.float64, device=dev)
        fv = capi.FvMatrix(mat, 1, dg, b, psi, V, ic, bcf)
        kw = dict(tolerance=0.0, maxIter=19)
        for name, fn in (("lduMatrix solve, 20 PCG iterations", lambda: mat.solve("PCG", "DIC", psi, b, **kw)),
                         ("fvMatrix::solve, 20 PCG iterations", lambda: fv.solve("PCG", "DIC", **kw))):
            psi.zero_()
            timeit(name, 20 * (160 * N + 32 * F), fn)
    except Exception as e:  # noqa: BLE001 -- keep the table above
        fvm_error = repr(e)
        print("fvMatrix glue:", fvm_error, file=sys.stderr)
    solves["fvMatrix_glue_error"] = fvm_error
    print(json.dumps({"n": n, "peak_gbs": peak, "peak_source": peak_src, "pcg_sweeps": sweeps, "kernels": rows,
                      "solves": solves}))
    addr.close()
    ctx.close()


if __name__ == "__main__":
    main()
