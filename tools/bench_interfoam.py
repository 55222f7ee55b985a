"""The face passes of the interFoam phase-fraction step on the device, timed: b200ldu_fv_limited_flux against the four calls it
replaces (limiter, limited weights, interpolation, product), b200ldu_vof_interface_flux against its composition of field operators,
alternating in the same run, and one alphaEqn corrector (explicit branch, vanLeer + compression) with the fused passes and with
the compositions.  Needs a GPU; bytes are the algorithm's, computed from the shapes.
  python tools/bench_interfoam.py [--n 256] [--reps 20]   -> one JSON line"""
import argparse
import importlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=256)
ap.add_argument("--reps", type=int, default=20)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_interfoam: no CUDA device -- timings come from the GPU only")
capi = importlib.import_module("rapidcfd-dev_b200.capi")
itf = importlib.import_module("rapidcfd-dev_b200.interfoam")
mules = importlib.import_module("rapidcfd-dev_b200.mules")
meshmod = importlib.import_module("rapidcfd-dev_b200.mesh")
import interfoam_cases as ic  # noqa: E402  (the sphere, the rotating flux and the mesh arrays of the tests)

ctx = capi.Context(0)
m = meshmod.hex_mesh(args.n)
mesh = itf.Mesh(capi, ctx, torch, **ic.geometry(m))
ph = itf.Phase(mesh, ic.sphere(m, width=1.5))
mix = itf.InterfaceProperties(capi, mesh, ph.alpha1, 1.0, 0.07)
phiH, dt = ic.rotation_flux(m)
phi, o, a = mesh.t(phiH), mesh.ops, mesh.addr
N, F, B = mesh.n, mesh.nF, mesh.nB
SCHEME = ("vanLeer", 1.0)


def flux_fused(flux, vf, g):
    return capi.fv_limited_flux(a, SCHEME[0], flux, vf, g, mesh.C, mesh.w, SCHEME[1])


def flux_composed(flux, vf, g):
    w = capi.fv_limited_weights(ctx, flux, capi.fv_limiter(a, SCHEME[0], flux, vf, g, mesh.C, SCHEME[1]), mesh.w)
    return o.mul(flux, capi.fv_interpolate_linear(a, 1, w, vf))


def iface_fused():
    return capi.vof_interface_flux(a, mesh.w, mix.gradAlpha, mesh.Sf, mesh.bSf, mesh.zeroB, mesh.deltaN, phi, mesh.magSf, 1.0)


def iface_composed():
    """the internal faces of the same expression through the field operators (the boundary pass has no counterpart to time)"""
    gf = capi.fv_interpolate_linear(a, 3, mesh.w, mix.gradAlpha)
    den = o.sadd(torch.sqrt(o.dot3(gf, gf)), mesh.deltaN)      # torch.sqrt: the operator set has no root; timing only
    nHatf = o.dot3(o.div(gf, den, 3, 1), mesh.Sf)
    return nHatf, o.mul(o.smul(1.0, o.mag(o.div(phi, mesh.magSf))), nHatf)


def corrector(flux):
    """one pass of the alphaEqn.H corrector loop, explicit branch, with `flux` for the three fvc::flux"""
    phir = iface_fused()[2]
    g1, g2 = mix.gradAlpha, mesh.grad(ph.alpha2, o.gather(mesh.bfc, ph.alpha2))
    phirb = o.neg(flux(o.neg(phir), ph.alpha2, g2))
    un = o.add(flux(phi, ph.alpha1, g1), flux(phirb, ph.alpha1, g1))
    aB = o.gather(mesh.bfc, ph.alpha1)
    lim, limB = mules.limit(capi, a, o, mesh.V, 1 / dt, ph.alpha1, ph.alpha1, aB, phi, mesh.zeroB, un, mesh.zeroB, 1.0, 0.0, 3)
    return mules.explicit_solve(capi, a, o, mesh.V, 1 / dt, ph.alpha1, lim, limB)


def timed(pairs, reps):
    """alternates the candidates inside one timed loop; ms per call, median over the repetitions"""
    ev = lambda: torch.cuda.Event(enable_timing=True)
    out = {k: [] for k in pairs}
    for k, f in pairs.items():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    for _ in range(reps):
        for k, f in pairs.items():
            e0, e1 = ev(), ev()
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            out[k].append(e0.elapsed_time(e1))
    return {k: float(np.median(v)) for k, v in out.items()}


g1 = mix.gradAlpha
assert torch.equal(flux_fused(phi, ph.alpha1, g1), flux_composed(phi, ph.alpha1, g1))
assert torch.equal(corrector(flux_fused), corrector(flux_composed))
t = timed({"limited_flux fused": lambda: flux_fused(phi, ph.alpha1, g1), "limited_flux 4 calls": lambda: flux_composed(phi, ph.alpha1, g1),
           "interface_flux fused": iface_fused, "interface_flux field operators": iface_composed,
           "corrector fused": lambda: corrector(flux_fused), "corrector 4-call fluxes": lambda: corrector(flux_composed)}, args.reps)
# algorithmic bytes, from the shapes: per face flux, cd weight, result (8 B each) and owner + neighbour (4 B each); per cell vf (8),
# gradc (24) and C (24), each cell read once.  The composition also writes and reads back limiter, weights and face value: 3 x 16 B/face.
bytes_flux = F * (8 + 8 + 8 + 8) + N * 56
bytes_flux_composed = bytes_flux + 3 * 16 * F
# interface flux with phi: per face w, phi, magSf, nHatf, phir (8 each), Sf (24), owner + neighbour (8); per cell gradAlpha (24);
# per boundary face cell index (4), bSf (24), snGrad (8), nHatfB (8) and a gathered gradient (24)
bytes_iface = F * (5 * 8 + 24 + 8) + N * 24 + B * (4 + 24 + 8 + 8 + 24)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"workload": f"interFoam alphaEqn face passes, {args.n}^3 hex cells, vanLeer, median of {args.reps}", "gpu": q,
                  "ms": {k: round(v, 4) for k, v in t.items()},
                  "algorithmic_GB": {"limited_flux": bytes_flux / 1e9, "limited_flux 4 calls": bytes_flux_composed / 1e9,
                                     "interface_flux": bytes_iface / 1e9},
                  "algorithmic_GBps": {"limited_flux fused": bytes_flux / t["limited_flux fused"] / 1e6,
                                       "limited_flux 4 calls": bytes_flux_composed / t["limited_flux 4 calls"] / 1e6,
                                       "interface_flux fused": bytes_iface / t["interface_flux fused"] / 1e6}}))
mesh.close()
ctx.close()
