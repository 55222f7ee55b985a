"""b200ldu_fv_limited_flux, b200ldu_vof_interface_flux and the phase-fraction step of rapidcfd-dev_b200/interfoam.py on the device
against the oracle (bit for bit where every piece is), against the four-call composition the fused flux replaces, against the
golden vectors, and a 64^3 rotation with compression: bounded, conservative, sharper than without."""
import importlib
import os

import numpy as np
import pytest

import interfoam_cases as ic
from oracle import interfoam_oracle as io
from oracle import limiters_oracle as lo
from test_interfoam_cpu import _fields

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def gpu():
    import torch
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


def _case(capi, ctx, torch, meshmod, seed):
    m = meshmod.hex_mesh(11, 9, 8)
    _, bfc = m.patch_start_facecells(m.wall_patches())
    addr = capi.mesh_to_device(ctx, m)
    capi.fv_boundary_set(addr, bfc)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64).ravel()).to(ctx.device)
    return m, bfc, addr, t, _fields(m, seed)


@pytest.mark.parametrize("scheme", sorted(lo.SCHEMES))
def test_limited_flux_on_the_device(gpu, meshmod, scheme):
    capi, ctx, torch = gpu
    m, bfc, addr, t, d = _case(capi, ctx, torch, meshmod, 31)
    ops = capi.FieldOps(ctx)
    flux, vf, g, C, cd = (t(d[k]) for k in ("flux", "vf", "g", "C", "cd"))
    for k in ((1.0, 0.3) if scheme == "limitedLinear" else (1.0,)):
        for fs, os_ in ((1, 1), (-1, -1), (-1, 1), (1, -1)):
            got = capi.fv_limited_flux(addr, scheme, flux, vf, g, C, cd, k, fs, os_).cpu().numpy()
            assert np.array_equal(got, io.limited_flux(scheme, m.lower, m.upper, d["flux"], d["vf"], d["g"], d["C"], d["cd"], k, fs, os_))
            # the four ABI calls it replaces, with the sign changes as field operations
            F = ops.neg(flux) if fs < 0 else flux
            w = capi.fv_limited_weights(ctx, F, capi.fv_limiter(addr, scheme, F, vf, g, C, k), cd)
            comp = ops.mul(F, capi.fv_interpolate_linear(addr, 1, w, vf))
            assert np.array_equal(got, (ops.neg(comp) if os_ < 0 else comp).cpu().numpy()), (k, fs, os_)
    addr.close()


def test_interface_flux_and_curvature_on_the_device(gpu, meshmod, orc):
    capi, ctx, torch = gpu
    m, bfc, addr, t, d = _case(capi, ctx, torch, meshmod, 32)
    rng = np.random.default_rng(33)
    bSf, bSn, V = rng.uniform(-1, 1, (len(bfc), 3)), rng.uniform(-1, 1, len(bfc)), rng.uniform(0.5, 2, m.nCells)
    bSn[::3] = 0.0
    a = orc.Addr(m.nCells, m.lower, m.upper)
    for deltaN in (1e-7, 0.5):
        for withPhi in (False, True):
            nHatf, nHatfB, phir = capi.vof_interface_flux(addr, t(d["w"]), t(d["g"]), t(d["Sf"]), t(bSf), t(bSn), deltaN,
                                                          t(d["flux"]) if withPhi else None, t(d["magSf"]) if withPhi else None, 0.75)
            w0, w1, w2 = io.interface_flux(m.lower, m.upper, d["w"], d["g"], d["Sf"], bfc, bSf, bSn, deltaN, d["flux"] if withPhi else None,
                                           d["magSf"], 0.75)
            assert np.array_equal(nHatf.cpu().numpy(), w0) and np.array_equal(nHatfB.cpu().numpy(), w1)
            assert (phir is None) if not withPhi else np.array_equal(phir.cpu().numpy(), w2)
        K = capi.FieldOps(ctx).neg(capi.fv_surface_integrate(addr, 1, nHatf, nHatfB, t(V), True, -1))
        assert np.array_equal(K.cpu().numpy(), -np.asarray(orc.surface_integrate(a, w0, bfc, w1, V, 1, True, -1)))
    addr.close()


def test_argument_errors_are_status_codes(gpu, meshmod):
    capi, ctx, torch = gpu
    m, bfc, addr, t, d = _case(capi, ctx, torch, meshmod, 34)
    flux, vf, g, C, cd = (t(d[k]) for k in ("flux", "vf", "g", "C", "cd"))
    with pytest.raises(capi.B200LduError, match="Unknown discretisation scheme QUICK"):
        capi.fv_limited_flux(addr, "QUICK", flux, vf, g, C, cd)
    with pytest.raises(capi.B200LduError):
        capi.fv_limited_flux(addr, "limitedLinear", flux, vf, g, C, cd, k=1.5)
    with pytest.raises(capi.B200LduError):
        capi.fv_limited_flux(addr, "vanLeer", flux, vf, None, C, cd)         # a limited scheme needs the gradient
    with pytest.raises(capi.B200LduError):
        capi.fv_limited_flux(addr, "upwind", flux, vf, None, None, cd, fluxSign=2)
    with pytest.raises(capi.B200LduError):
        capi.vof_interface_flux(addr, t(d["w"]), None, t(d["Sf"]), t(np.zeros((len(bfc), 3))), t(np.zeros(len(bfc))), 1e-7)
    with pytest.raises(capi.B200LduError):
        capi.vof_interface_flux(addr, t(d["w"]), t(d["g"]), t(d["Sf"]), t(np.ones((len(bfc), 3))), t(np.zeros(len(bfc))), 1e-7, flux, None, 1.0)
    assert capi.fv_limited_flux(addr, "upwind", flux, vf, None, None, cd).numel() == m.nFaces    # upwind and linear need neither
    addr.close()


@pytest.mark.parametrize("MULESCorr", [False, True])
def test_step_against_the_oracle_and_the_golden_vectors(gpu, meshmod, orc, MULESCorr):
    capi, ctx, torch = gpu
    m = meshmod.hex_mesh(12)
    a0 = ic.sphere(m)
    ctl = ic.controls(MULESCorr, 2, 2)
    mesh, mix, ph = ic.run_product(capi, ctx, torch, m, a0, ctl, 3, ic.SOLVER)
    o = ic.run_oracle(orc, m, a0, ctl, 3, ic.SOLVER)
    got = {k: getattr(ph, k).cpu().numpy() for k in ("alpha1", "alpha2", "rhoPhi", "rhoPhiB", "rho")}
    got.update(K=mix.K.cpu().numpy(), nHatf=mix.nHatf.cpu().numpy(), stf=mix.surface_tension_force().cpu().numpy())
    want = dict(alpha1=o.alpha1, alpha2=o.alpha2, rhoPhi=o.rhoPhi, rhoPhiB=o.rhoPhiB, rho=o.rho, K=o.K, nHatf=o.nHatf, stf=o.surface_tension_force())
    for k in ("alpha1", "alpha2", "rhoPhi", "rhoPhiB", "rho"):
        if MULESCorr:   # one linear solve per pass
            assert np.allclose(got[k], want[k], rtol=0, atol=1e-9 * max(1.0, np.abs(want[k]).max())), k
        else:           # every piece is bit-exact on its own
            assert np.array_equal(got[k], want[k]), k
    if not MULESCorr:
        for k in ("K", "nHatf", "stf"):
            assert np.array_equal(got[k], want[k]), k
    assert np.allclose(ph.reports, o.reports, rtol=0, atol=1e-9)
    mesh.close()
    # the golden vectors: the state of the sphere on 10^3 cells, and two steps with two correctors
    gold = np.load(os.path.join(HERE, "golden", "interfoam_golden.npz"))
    mg = meshmod.hex_mesh(10)
    mesh, mix, ph = ic.run_product(capi, ctx, torch, mg, ic.sphere(mg), ic.controls(MULESCorr, 2, 1), 0)
    assert np.array_equal(mix.nHatf.cpu().numpy(), gold["nHatf"]) and np.array_equal(mix.nHatfB.cpu().numpy(), gold["nHatfB"])
    assert np.array_equal(mix.K.cpu().numpy(), gold["K"])
    assert np.array_equal(mix.compression_flux(mesh.t(ic.rotation_flux(mg)[0])).cpu().numpy(), gold["phir"])
    mesh.close()
    mesh, mix, ph = ic.run_product(capi, ctx, torch, mg, ic.sphere(mg), ic.controls(MULESCorr, 2, 1), 2, ic.SOLVER)
    if MULESCorr:
        assert np.allclose(ph.alpha1.cpu().numpy(), gold["alpha_mulescorr"], rtol=0, atol=1e-9)
    else:
        assert np.array_equal(ph.alpha1.cpu().numpy(), gold["alpha_explicit"])
    mesh.close()


def test_rotation_64_cubed_with_compression(gpu, meshmod):
    capi, ctx, torch = gpu
    m = meshmod.hex_mesh(64)
    a0, V = ic.sphere(m, width=1.5), m.volumes()
    out = {}
    for cAlpha in (0.0, 1.0):
        mesh, mix, ph = ic.run_product(capi, ctx, torch, m, a0, ic.controls(cAlpha=cAlpha), 10)
        out[cAlpha] = ph.alpha1.cpu().numpy()
        assert torch.isfinite(mix.K).all()
        mesh.close()
    for a in out.values():
        assert a.min() >= -1e-10 and a.max() <= 1 + 1e-10
        assert abs((a * V).sum() - (a0 * V).sum()) <= 1e-11 * (a0 * V).sum()
    assert ic.band(out[1.0]) < ic.band(out[0.0])
