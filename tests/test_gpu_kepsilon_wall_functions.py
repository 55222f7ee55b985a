"""The k-epsilon wall functions on the device: fvMatrix::setValues, nutkWallFunction and epsilonWallFunction entry points against
oracle/wallfn_oracle.py, and three kEpsilon::correct() calls with kqRWallFunction / epsilonWallFunction / nutkWallFunction walls in
lockstep with wallfn_oracle.KEpsilonWall (the harness of tests/test_gpu_step_lockstep.py: every solved system bit for bit, every
field between the solves bit for bit, every solution within the true-residual bound of DESIGN.md section 2).

Values through log (nutk) and pow (epsilon0) may differ from the C library's in the last bits: CUDA's log and pow are within 1 and
2 ulp.  Those are held to WALLFN_REL; everything else is compared bit for bit.  In the lockstep runs the oracle checks its own wall
values against the product's the same way (bit for bit on the stand-in) and then goes on from the product's, as it does with each
solution, so that every solved system and every field can still be compared bit for bit."""
import importlib

import numpy as np
import pytest

import polymesh_cases as pc
import wallfn_backend
from oracle import fvm_oracle as fo
from oracle import piso_oracle as po
from oracle import wallfn_oracle as wo
from test_gpu_engine_streams import Mismatches
from test_gpu_step_lockstep import CTL, Lockstep, _ke_snap, host

WALLFN_REL = 1e-15
BACKENDS = ["stand-in", pytest.param("device", marks=pytest.mark.gpu)]


@pytest.fixture(scope="module", params=BACKENDS)
def backend(request):
    if request.param == "stand-in":
        yield wallfn_backend.fixture()
        return
    import torch
    assert torch.cuda.is_available()
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    ctx = capi.Context(0)
    yield capi, ctx, torch
    ctx.close()


def _ff():
    return importlib.import_module("rapidcfd-dev_b200.foamfile")


# ---- the cases ------------------------------------------------------------------------------------------------------------------
def cavity_walls(meshmod, n):
    """the n^3 cavity's six patches: five walls with wall functions, the last one fixedValue for k, epsilon and nut"""
    m = meshmod.hex_mesh(n)
    ps = np.concatenate([[0], np.cumsum([len(p.faceCells) for p in m.patches])])
    nP = len(m.patches)
    types = dict(kTypes=["kqRWallFunction"] * (nP - 1) + ["fixedValue"], epsTypes=["epsilonWallFunction"] * (nP - 1) + ["fixedValue"],
                 nutTypes=["nutkWallFunction"] * (nP - 1) + ["fixedValue"])
    y = _ff().from_hex_mesh(m).near_wall_dist([p.name for p in m.patches])
    return m, ps, types, y


def kepsilon_wall_case(meshmod, orc, n=10, divScheme="upwind", alpha=None):
    m, ref = po.cavity_from_hex(orc, meshmod, n)
    m, ps, types, y = cavity_walls(meshmod, n)
    nB = len(ref.bfc)
    bMagSf, bDelta = np.full(nB, m.h * m.h), np.full(nB, 2.0 / m.h)
    kB, eB = np.full(nB, 0.015), np.full(nB, 0.08)
    rng = np.random.default_rng(21)
    k0, e0 = rng.uniform(0.01, 0.02, m.nCells), rng.uniform(0.05, 0.1, m.nCells)
    low = ref.bfc[ps[2]:ps[3]]                   # a band of large k over one wall: yPlus above yPlusLam there, below elsewhere
    k0[low] = rng.uniform(20.0, 60.0, len(low))
    flow = {}

    def product(capi, ctx, torch, L):
        ico = importlib.import_module("rapidcfd-dev_b200.icofoam")
        kem = importlib.import_module("rapidcfd-dev_b200.kepsilon")
        _, case = ico.cavity(capi, ctx, torch, n)
        L.paused = True
        for _ in range(3):
            case.step(UControls=CTL, pControls=CTL)
        L.paused = False
        flow.update(U=host(case.U).reshape(-1, 3), phi=host(case.phi), bphi=host(case.bphi), deltaT=case.deltaT)
        ke = kem.KEpsilon(capi, case, bMagSf, bDelta, k0, e0, kB, eB, patchStart=ps, y=y, **types)
        snaps = [_ke_snap(m, ke, True)]
        for _ in range(3):
            ke.correct(case.U, case.phi, case.bphi, case.deltaT, divScheme, alpha, alpha, controls=CTL)
            snaps.append(_ke_snap(m, ke, True))
        ke.close()
        case.close()
        return snaps

    def oracle():
        ke = wo.KEpsilonWall(orc, ref.addr, ref.Sf, ref.magSf, ref.w, ref.delta, ref.V, ref.bfc, ref.bSf, bMagSf, bDelta, ref.Ub, ref.nu, k0,
                             e0, kB, eB, ps, types["kTypes"], types["epsTypes"], types["nutTypes"], y)
        snaps = [_ke_snap(m, ke, False)]
        for _ in range(3):
            ke.correct(flow["U"], flow["phi"], flow["bphi"], flow["deltaT"], divScheme, alpha, alpha, controls=CTL)
            snaps.append(_ke_snap(m, ke, False))
        return snaps

    return product, oracle, (ref.bfc, ps)


def kepsilon_wall_polymesh_case(orc):
    """the split-hex box (rows with up to 24 faces per side, cells on up to three walls): every patch a wall with wall functions"""
    b = pc.refined_box(5, "random", seed=7)
    C, nB = b.cell_centres(), len(b.bFaceCells)
    U, Ub, phi = pc.velocity(C), pc.velocity(b.bCf), pc.solenoidal_flux(b)
    bphi, deltaT, nu = np.zeros(nB), 0.02, 0.01
    geo = (b.nCells, b.lower, b.upper, b.Sf(), b.magSf(), b.weights(), b.deltaCoeffs(), b.volumes(), b.bFaceCells, b.bSf, b.bMagSf(),
           b.bDeltaCoeffs(), Ub, nu, deltaT)
    walls = b.wall_patches()
    ps = np.concatenate([[0], np.cumsum([len(p.faceCells) for p in walls])])
    nP = len(walls)
    types = dict(kTypes=["kqRWallFunction"] * nP, epsTypes=["epsilonWallFunction"] * nP, nutTypes=["nutkWallFunction"] * nP)
    y = b.pm.near_wall_dist([p.name for p in walls])
    rng = np.random.default_rng(23)
    k0, e0 = rng.uniform(0.01, 0.02, b.nCells), rng.uniform(0.05, 0.1, b.nCells)
    k0[b.bFaceCells[::3]] = rng.uniform(20.0, 60.0, len(b.bFaceCells[::3]))
    kB, eB = np.full(nB, 0.015), np.full(nB, 0.08)

    def product(capi, ctx, torch, L):
        ico = importlib.import_module("rapidcfd-dev_b200.icofoam")
        kem = importlib.import_module("rapidcfd-dev_b200.kepsilon")
        case = ico.IcoFoam(capi, ctx, torch, *geo, cellCentres=C)
        case.U, case.phi, case.bphi = case._t(U), case._t(phi), case._t(bphi)
        ke = kem.KEpsilon(capi, case, b.bMagSf(), b.bDeltaCoeffs(), k0, e0, kB, eB, patchStart=ps, y=y, **types)
        snaps = [_ke_snap(None, ke, True)]
        for divScheme, alpha in (("upwind", None), ("linear", 0.7), ("linear", None)):
            ke.correct(case.U, case.phi, case.bphi, deltaT, divScheme, alpha, alpha, controls=CTL)
            snaps.append(_ke_snap(None, ke, True))
        ke.close()
        case.close()
        return snaps

    def oracle():
        ref = po.Cavity(orc, *geo)
        ke = wo.KEpsilonWall(orc, ref.addr, ref.Sf, ref.magSf, ref.w, ref.delta, ref.V, ref.bfc, ref.bSf, b.bMagSf(), b.bDeltaCoeffs(),
                             ref.Ub, nu, k0, e0, kB, eB, ps, types["kTypes"], types["epsTypes"], types["nutTypes"], y)
        snaps = [_ke_snap(None, ke, False)]
        for divScheme, alpha in (("upwind", None), ("linear", 0.7), ("linear", None)):
            ke.correct(U, phi, bphi, deltaT, divScheme, alpha, alpha, controls=CTL)
            snaps.append(_ke_snap(None, ke, False))
        return snaps

    return product, oracle, (b.bFaceCells, ps)


def check_wall_cells(L, bfc):
    """after each epsilon solve the wall cells hold epsilon0 -- the value setValues put into psi -- to rel 1e-12 (the cavity: every
    wall cell's last setValues leaves its row alone)"""
    wall = np.unique(bfc)
    for d in L.dev[0::2]:
        before, after = d["psi0"][wall], d["psi"][wall]
        assert np.all(np.abs(after - before) <= 1e-12 * np.abs(before)), np.max(np.abs(after - before) / np.abs(before))


# ---- lockstep ------------------------------------------------------------------------------------------------------------------
class WallValues:
    """the wall-function values of the product run (capi.wallfn_nutk / wallfn_epsilon outputs, in call order), handed to the oracle
    run in place of its own once they agree with them"""

    def __init__(self, monkeypatch, capi, device):
        self.mp, self.capi, self.device, self.rec, self.k, self.M = monkeypatch, capi, device, [], 0, Mismatches()

    def record(self):
        nutk0, eps0 = self.capi.wallfn_nutk, self.capi.wallfn_epsilon

        def nutk(addr, faces, y, k, nuw, yPlusLam, Cmu25, nutB, *a):
            nutk0(addr, faces, y, k, nuw, yPlusLam, Cmu25, nutB, *a)
            self.rec.append(("nutk", host(nutB)[host_i(faces)]))

        def eps(addr, cw, y, k, U, Ub, bDelta, nutB, nu, Cmu25, Cmu75, G, epsilon, epsB, *a):
            eps0(addr, cw, y, k, U, Ub, bDelta, nutB, nu, Cmu25, Cmu75, G, epsilon, epsB, *a)
            self.rec.append(("epsilon", (host(G), host(epsilon), host(epsB))))

        self.mp.setattr(self.capi, "wallfn_nutk", nutk)
        self.mp.setattr(self.capi, "wallfn_epsilon", eps)

    def _take(self, kind, own):
        i = self.k
        self.k += 1
        if i >= len(self.rec) or self.rec[i][0] != kind:
            self.M.true(False, f"wall call {i}: the oracle calls {kind}, the product {self.rec[i][0] if i < len(self.rec) else 'nothing'}")
            return own
        got = self.rec[i][1]
        for j, (a, b) in enumerate(zip(got if kind == "epsilon" else [got], own if kind == "epsilon" else [own])):
            if self.device:
                self.M.true(np.all(np.abs(a - b) <= WALLFN_REL * np.abs(b)), f"wall call {i} ({kind}[{j}]): beyond rel {WALLFN_REL}")
            else:
                self.M.bits(a, b, f"wall call {i} ({kind}[{j}])")
        return tuple(x.copy() for x in got) if kind == "epsilon" else got.copy()

    def replay(self):
        nutk0, eps0 = wo.nutk, wo.epsilon_wall
        self.mp.setattr(wo, "nutk", lambda *a, **kw: self._take("nutk", nutk0(*a, **kw)))
        self.mp.setattr(wo, "epsilon_wall", lambda *a, **kw: self._take("epsilon", eps0(*a, **kw)))

    def check(self):
        self.M.true(self.k == len(self.rec), f"the product made {len(self.rec)} wall calls, the oracle {self.k}")
        self.M.check()


def host_i(x):
    return x.detach().cpu().numpy().astype(np.int64)


def run_wall_lockstep(monkeypatch, backend, product, oracle):
    """run_lockstep of tests/test_gpu_step_lockstep.py with the product's wall values handed to the oracle (WallValues)"""
    capi, ctx, torch = backend
    L = Lockstep(monkeypatch, capi, ctx.device != "cpu")
    W = WallValues(monkeypatch, capi, ctx.device != "cpu")
    L.record()
    W.record()
    dev = product(capi, ctx, torch, L)
    L.replay()                       # undoes every patch of the product run
    W.replay()
    ora = oracle()
    L.finish(dev, ora)
    W.check()
    L.snaps = ora
    return L


@pytest.mark.parametrize("alpha", [None, 0.7])
@pytest.mark.parametrize("divScheme", ["upwind", "linear"])
def test_kepsilon_wall_functions_cavity_in_lockstep(monkeypatch, backend, meshmod, orc, divScheme, alpha):
    product, oracle, (bfc, ps) = kepsilon_wall_case(meshmod, orc, 10, divScheme, alpha)
    L = run_wall_lockstep(monkeypatch, backend, product, oracle)
    assert len(L.dev) == 6
    check_wall_cells(L, bfc[:ps[-2]])
    # both sides of yPlusLam were exercised
    nutB = np.concatenate([s["nutB"][:ps[-2]] for s in L.snaps])
    assert (nutB == 0).any() and (nutB > 0).any()


def test_kepsilon_wall_functions_polymesh_in_lockstep(monkeypatch, backend, orc):
    product, oracle, (bfc, ps) = kepsilon_wall_polymesh_case(orc)
    L = run_wall_lockstep(monkeypatch, backend, product, oracle)
    assert len(L.dev) == 6
    # no wall-cell check here: a wall cell set by one patch's setValues and not by a later one's has its source changed by the later
    # call wherever it neighbours a cell of the later patch only (the reference's unset-cell pass, DESIGN.md section 2)


# ---- the entry points one by one -------------------------------------------------------------------------------------------------
def _entry_case(meshmod, orc, seed=5):
    """a 6^3 hex mesh with an asymmetric matrix, random fields and the cavity's wall set-up"""
    m, ps, types, y = cavity_walls(meshmod, 6)
    bfc = np.concatenate([p.faceCells for p in m.patches]).astype(np.int32)
    n, nF, nB = m.nCells, len(m.lower), len(bfc)
    rng = np.random.default_rng(seed)
    r = lambda lo, hi, k: rng.uniform(lo, hi, k)
    k = r(0.01, 0.02, n)
    k[bfc[ps[1]:ps[2]]] = r(20.0, 60.0, ps[2] - ps[1])
    epsWall = np.repeat([t == "epsilonWallFunction" for t in types["epsTypes"]], np.diff(ps))
    return dict(m=m, ps=ps, bfc=bfc, y=y, n=n, diag=r(5, 6, n), upper=r(-1, 0, nF), lower=r(-1, 0, nF), source=r(-1, 1, n), psi=r(0, 1, n),
                ic=r(0, 1, nB), bc=r(0, 1, nB), k=k, U=r(-1, 1, 3 * n), Ub=r(-1, 1, 3 * nB), bDelta=np.full(nB, 2.0 / m.h), nutB=r(0, 1e-3, nB),
                G=r(0, 1, n), eps=r(0.05, 0.1, n), epsB=r(0.05, 0.1, nB), cw=wo.corner_weights(n, bfc, epsWall),
                nutkFaces=np.nonzero(np.repeat([t == "nutkWallFunction" for t in types["nutTypes"]], np.diff(ps)))[0].astype(np.int32))


def _oracle_entries(orc, c):
    a = orc.Addr(c["n"], c["m"].lower, c["m"].upper)
    om = fo.FvMatrix(orc, a, 1, c["diag"], c["upper"], c["lower"], c["source"], c["psi"], np.ones(c["n"]), c["bfc"], c["ic"], c["bc"])
    for p in (0, 2):                                     # two patches that share edge cells: the second call sees the first's clearing
        cells = c["bfc"][c["ps"][p]:c["ps"][p + 1]]
        wo.set_values(om, cells, om.psi[cells, 0].copy() * 0 + (p + 1.5))
    Cmu25, Cmu75 = wo.constants()
    f = c["nutkFaces"]
    nutB = c["nutB"].copy()
    nutB[f] = wo.nutk(c["y"][f], c["k"][c["bfc"][f]], 0.01, wo.y_plus_lam(), Cmu25)
    G, eps, epsB = wo.epsilon_wall(c["bfc"], c["cw"], c["y"], c["k"], c["U"], c["Ub"], c["bDelta"], c["nutB"], 0.01, c["G"], c["eps"], c["epsB"],
                                   Cmu25, Cmu75)
    return dict(psi=om.psi[:, 0], source=om.source[:, 0], upper=om.upper, lower=om.lower, ic=om.ic[:, 0], bc=om.bc[:, 0], nutB=nutB,
                G=G, eps=eps, epsB=epsB)


def _device_entries(capi, ctx, torch, c, guard=0):
    """the entry points on the device; guard > 0: every caller buffer lives inside a NaN-filled allocation, `guard` values each side"""
    dev = ctx.device
    keep = []

    def t(a, dtype=torch.float64):
        a = np.ascontiguousarray(a)
        full = torch.full((a.size + 2 * guard,), float("nan"), dtype=torch.float64, device=dev) if dtype == torch.float64 else \
            torch.full((a.size + 2 * guard,), -7, dtype=dtype, device=dev)
        full[guard:guard + a.size] = torch.from_numpy(a).to(dev)
        keep.append(full)
        return full[guard:guard + a.size]

    i32 = lambda a: t(np.asarray(a, np.int32), torch.int32)
    m = c["m"]
    addr = capi.mesh_to_device(ctx, m)
    capi.fv_boundary_set(addr, c["bfc"])
    mat = capi.LduMatrix(addr)
    diag, upper, lower, source, psi, ic, bc = (t(c[k]) for k in ("diag", "upper", "lower", "source", "psi", "ic", "bc"))
    mat.set(diag, upper, lower)
    eqn = capi.FvMatrix(mat, 1, diag, source, psi, t(np.ones(c["n"])), ic, bc)
    for p in (0, 2):
        cells = c["bfc"][c["ps"][p]:c["ps"][p + 1]]
        eqn.setValues(i32(cells), t(np.full(len(cells), p + 1.5)), upper, lower)
    Cmu25, Cmu75 = wo.constants()
    nutB = t(c["nutB"])
    capi.wallfn_nutk(addr, i32(c["nutkFaces"]), t(c["y"]), t(c["k"]), 0.01, wo.y_plus_lam(), Cmu25, nutB)
    G, eps, epsB = t(c["G"]), t(c["eps"]), t(c["epsB"])
    capi.wallfn_epsilon(addr, t(c["cw"]), t(c["y"]), t(c["k"]), t(c["U"]), t(c["Ub"]), t(c["bDelta"]), t(c["nutB"]), 0.01, Cmu25, Cmu75, G,
                        eps, epsB)
    out = {k: host(v) for k, v in dict(psi=psi, source=source, upper=upper, lower=lower, ic=ic, bc=bc, nutB=nutB, G=G, eps=eps,
                                          epsB=epsB).items()}
    if guard:
        for full in keep:
            h = full.cpu().numpy()
            edge = np.concatenate([h[:guard], h[-guard:]])
            assert (np.isnan(edge) if full.dtype == torch.float64 else edge == -7).all(), "a guard value was overwritten"
    mat.close()
    addr.close()
    return out


def _compare(M, got, ref):
    for k in ("psi", "source", "upper", "lower", "ic", "bc", "G"):
        M.bits(got[k], ref[k], k)
    for k in ("nutB", "eps", "epsB"):                # through log / pow: within WALLFN_REL of the C library's
        M.true(np.all(np.abs(got[k] - ref[k]) <= WALLFN_REL * np.abs(ref[k])), f"{k}: rel {np.max(np.abs(got[k] - ref[k]) / np.maximum(np.abs(ref[k]), 1e-300)):.2e}")


@pytest.mark.gpu
def test_wall_function_entry_points_match_the_oracle(meshmod, orc):
    import torch
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    c = _entry_case(meshmod, orc)
    ref = _oracle_entries(orc, c)
    ctx = capi.Context(0)
    got = _device_entries(capi, ctx, torch, c)
    ctx.close()
    M = Mismatches()
    _compare(M, got, ref)
    M.check()
    assert (got["nutB"][c["nutkFaces"]] == 0).any() and (got["nutB"][c["nutkFaces"]] > 0).any()


@pytest.mark.gpu
def test_wall_function_entry_points_under_poisoned_workspace(monkeypatch, meshmod, orc):
    """B200LDU_POISON_ALLOC=1 (every new workspace block NaN-filled) and NaN-guarded caller buffers: the same results, bit for bit,
    as a clean context, and nothing written outside the caller's arrays"""
    import torch
    capi = importlib.import_module("rapidcfd-dev_b200.capi")
    c = _entry_case(meshmod, orc, seed=9)
    ctx = capi.Context(0)
    clean = _device_entries(capi, ctx, torch, c)
    ctx.close()
    monkeypatch.setenv("B200LDU_POISON_ALLOC", "1")
    ctx = capi.Context(0)
    poisoned = _device_entries(capi, ctx, torch, c, guard=64)
    ctx.close()
    M = Mismatches()
    for k in clean:
        M.bits(poisoned[k], clean[k], k)
    M.check()
