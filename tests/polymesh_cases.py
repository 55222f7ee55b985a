"""Meshes whose cells have more faces than a hex box gives them, for the tests of the cell-walking kernels (fv_kernels.cuh,
fvmatrix_kernels.cuh, mules_kernels.cuh, vof_kernels.cuh), the asymmetric engine and GAMG.

refined_box(n, order): an n^3 lattice on the unit cube with every coarse cell of odd i+j+k split 2x2x2 (a checkerboard), the split
hexes snappyHexMesh leaves at a refinement interface.  Every face is one square of the (2n+1)^3 point lattice, except the boundary
faces of unsplit cells, which keep their edge midpoints (hanging points: a planar face keeps its area and centroid).  An interior
unsplit cell has 24 faces to 24 distinct fine cells, so no (owner, neighbour) pair repeats; `order` puts the unsplit cells first
(up to 24 owner faces), last (up to 24 losort faces) or in a seeded random order.  With `split_boundary` the z-min face of an
unsplit cell is four faces over two interleaved patches; with `periodic_x` (n odd) x-min and x-max are a cyclic pair of split
faces, four coupled faces per unsplit cell.

graph(n, k, seed): the random graph of tests/test_fv_kernels_cpu.py with random geometry, cells without any face and an unsorted
boundary list with several faces per cell.

Both return a PolyBox: the attributes the hex-mesh builders read (nCells, lower, upper, cell_centres(), Sf(), wall_patches(), ...).
Each generator asserts the face counts it exists for, so that a later change cannot quietly weaken a case."""
import importlib
from dataclasses import dataclass

import numpy as np

ff = importlib.import_module("rapidcfd-dev_b200.foamfile")

ORDERS = ("coarse-first", "fine-first", "random")


@dataclass
class BPatch:
    name: str
    faceCells: np.ndarray      # int32
    Sf: np.ndarray             # (P,3) outward
    Cf: np.ndarray             # (P,3)
    kind: str = "wall"         # wall | cyclic
    neighbRank: int = -1       # cyclic: -(partner index among the coupled patches + 1)


class PolyBox:
    """LDU view of a mesh with its finite-volume geometry (internal faces first, then the patches)"""

    def __init__(self, nCells, lower, upper, C, V, Sf, Cf, weights, deltaCoeffs, patches, pm=None):
        self.nCells, self.lower, self.upper = int(nCells), np.asarray(lower, np.int32), np.asarray(upper, np.int32)
        self.nFaces = len(self.lower)
        self._C, self._V, self._Sf, self._Cf, self._w, self._dc = C, V, Sf, Cf, weights, deltaCoeffs
        self.patches, self.pm = patches, pm
        walls = self.wall_patches()
        self.bFaceCells = np.concatenate([p.faceCells for p in walls]).astype(np.int32) if walls else np.zeros(0, np.int32)
        self.bSf = np.concatenate([p.Sf for p in walls]) if walls else np.zeros((0, 3))
        self.bCf = np.concatenate([p.Cf for p in walls]) if walls else np.zeros((0, 3))

    def cell_centres(self):
        return self._C

    def volumes(self):
        return self._V

    def Sf(self):
        return self._Sf

    def magSf(self):
        return np.sqrt((self._Sf ** 2).sum(1))

    def face_centres(self):
        return self._Cf

    def weights(self):
        return self._w

    def deltaCoeffs(self):
        return self._dc

    def bMagSf(self):
        return np.sqrt((self.bSf ** 2).sum(1))

    def bDeltaCoeffs(self):
        """1/|d.n| from the cell centre to the boundary face (the fixedValue gradient coefficient)"""
        n = self.bSf / self.bMagSf()[:, None]
        return 1.0 / np.abs(((self.bCf - self._C[self.bFaceCells]) * n).sum(1))

    def wall_patches(self):
        return [p for p in self.patches if p.kind == "wall"]

    def coupled_patches(self):
        return [p for p in self.patches if p.kind == "cyclic"]

    def patch_start_facecells(self, patches=None):
        ps = self.coupled_patches() if patches is None else patches
        start = np.zeros(len(ps) + 1, dtype=np.int32)
        for i, p in enumerate(ps):
            start[i + 1] = start[i] + len(p.faceCells)
        fc = np.concatenate([p.faceCells for p in ps]).astype(np.int32) if ps else np.zeros(0, np.int32)
        return start, fc

    def coupled_arrays(self):
        """(patchStart, faceCells, neighbRank, partner cell of every coupled face) or Nones without coupled patches"""
        cps = self.coupled_patches()
        if not cps:
            return None, None, None, None
        ps, fc = self.patch_start_facecells()
        nr = np.array([p.neighbRank for p in cps], np.int32)
        partner = np.concatenate([cps[-p.neighbRank - 1].faceCells for p in cps]).astype(np.int32)
        return ps, fc, nr, partner

    def counts(self):
        """faces per cell: owner, losort, non-coupled boundary, coupled; and the number of cells whose boundary faces lie in
        two or more patches"""
        n = self.nCells
        own, nei = np.bincount(self.lower, minlength=n), np.bincount(self.upper, minlength=n)
        bnd = np.bincount(self.bFaceCells, minlength=n)
        _, cfc = self.patch_start_facecells()
        cpl = np.bincount(cfc, minlength=n) if len(cfc) else np.zeros(n, int)
        patchesOf = [set() for _ in range(n)]
        for i, p in enumerate(self.wall_patches()):
            for c in np.unique(p.faceCells):
                patchesOf[c].add(i)
        multi = sum(len(s) >= 2 for s in patchesOf)
        return dict(owner=own, losort=nei, boundary=bnd, coupled=cpl, multiPatchCells=multi)


# ---- refined_box ---------------------------------------------------------------------------------------------------------
_PAIR = [(1, 2), (2, 0), (0, 1)]          # right-handed: e_a x e_b = e_axis


def _square(N, axis, plane, u, v):
    """point labels of the unit square at `plane` on `axis`, lower corner (u, v) in the other two axes, normal +axis"""
    a, b = _PAIR[axis]
    pts = []
    for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
        q = [0, 0, 0]
        q[axis], q[a], q[b] = plane, u + du, v + dv
        pts.append(q[0] + (N + 1) * (q[1] + (N + 1) * q[2]))
    return np.stack(pts, -1)


def _coarse_square(N, axis, plane, u, v):
    """the 2x2 square with its edge midpoints (8 points), lower corner (u, v), normal +axis"""
    a, b = _PAIR[axis]
    pts = []
    for du, dv in ((0, 0), (1, 0), (2, 0), (2, 1), (2, 2), (1, 2), (0, 2), (0, 1)):
        q = [0, 0, 0]
        q[axis], q[a], q[b] = plane, u + du, v + dv
        pts.append(q[0] + (N + 1) * (q[1] + (N + 1) * q[2]))
    return pts


def refined_box(n, order="coarse-first", split_boundary=True, periodic_x=False, seed=0):
    assert order in ORDERS and n >= 4
    assert not periodic_x or n % 2 == 1, "x-min and x-max split alike only for odd n"
    N = 2 * n
    c = np.arange(n ** 3)
    ci, cj, ck = c % n, (c // n) % n, c // (n * n)
    split = (ci + cj + ck) % 2 == 1
    nU, nS = int((~split).sum()), int(split.sum())
    nCells = nU + 8 * nS
    uid, fid = np.full(n ** 3, -1), np.full((n ** 3, 8), -1)
    if order == "fine-first":
        fid[split] = np.arange(8 * nS).reshape(nS, 8)
        uid[~split] = 8 * nS + np.arange(nU)
    else:
        uid[~split] = np.arange(nU)
        fid[split] = nU + np.arange(8 * nS).reshape(nS, 8)
    if order == "random":
        perm = np.random.default_rng(seed).permutation(nCells)
        uid[~split], fid[split] = perm[uid[~split]], perm[fid[split]]
    # voxel (fine lattice cell) -> mesh cell
    a, b, cc = np.meshgrid(np.arange(N), np.arange(N), np.arange(N), indexing="ij")
    coarse = a // 2 + n * (b // 2 + n * (cc // 2))
    child = a % 2 + 2 * (b % 2) + 4 * (cc % 2)
    vox = np.where(split[coarse], fid[coarse, child], uid[coarse])
    isUnsplit = np.zeros(nCells, bool)
    isUnsplit[uid[~split]] = True

    # internal faces: one lattice square between two voxels of different cells
    own, nei, quads = [], [], []
    for axis in range(3):
        sl0, sl1 = [slice(None)] * 3, [slice(None)] * 3
        sl0[axis], sl1[axis] = slice(0, N - 1), slice(1, N)
        A, B = vox[tuple(sl0)], vox[tuple(sl1)]
        keep = A != B
        idx = np.nonzero(keep)
        pa, pb_ = _PAIR[axis]
        q = _square(N, axis, idx[axis] + 1, idx[pa], idx[pb_])
        lo, hi = np.minimum(A[keep], B[keep]), np.maximum(A[keep], B[keep])
        q = np.where((A[keep] == lo)[:, None], q, q[:, ::-1])         # normal from owner to neighbour
        own.append(lo), nei.append(hi), quads.extend(list(q))
    own, nei = np.concatenate(own), np.concatenate(nei)
    o = np.lexsort((nei, own))
    own, nei = own[o], nei[o]
    quads = [quads[i] for i in o]
    assert len(np.unique(own.astype(np.int64) * nCells + nei)) == len(own), "an (owner, neighbour) pair repeats"

    # boundary faces, patch by patch
    def side(axis, hi, merge):
        """(cells, faces) of one side, ordered by position; unsplit cells' four squares merged when `merge`"""
        pa, pb_ = _PAIR[axis]
        layer = N - 1 if hi else 0
        plane = N if hi else 0
        out = []
        for v in range(N):
            for u in range(N):
                q = [0, 0, 0]
                q[axis], q[pa], q[pb_] = layer, u, v
                cell = vox[q[0], q[1], q[2]]
                if merge and isUnsplit[cell]:
                    if u % 2 or v % 2:
                        continue
                    pts = _coarse_square(N, axis, plane, u, v)
                else:
                    pts = list(_square(N, axis, plane, u, v))
                out.append((cell, (u, v), pts if hi else pts[::-1]))
        return out

    sides = [("xmin", 0, 0), ("xmax", 0, 1), ("ymin", 1, 0), ("ymax", 1, 1), ("zmin", 2, 0), ("zmax", 2, 1)]
    bpatches = []       # (name, type, [(cell, pts)])
    for name, axis, hi in sides:
        if axis == 0 and periodic_x:
            faces = side(axis, hi, False)
            bpatches.append((name, "cyclic", [(f[0], f[2]) for f in faces]))
        elif name == "zmin" and split_boundary:
            faces = side(axis, hi, False)
            for par in (0, 1):           # two patches, interleaved like a chequerboard
                bpatches.append((f"zmin{par}", "wall", [(f[0], f[2]) for f in faces if (f[1][0] + f[1][1]) % 2 == par]))
        else:
            bpatches.append((name, "wall", [(f[0], f[2]) for f in side(axis, hi, True)]))
    owner = [own]
    polys = list(quads)
    patches, start = [], len(own)
    for name, typ, faces in bpatches:
        owner.append(np.array([f[0] for f in faces], np.int32))
        polys.extend([np.asarray(f[1]) for f in faces])
        nb = ("xmax" if name == "xmin" else "xmin") if typ == "cyclic" else ""
        patches.append(ff.PolyPatch(name, typ, len(faces), start, neighbourPatch=nb))
        start += len(faces)
    sizes = np.array([len(p) for p in polys])
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    g = np.arange(N + 1) / N
    P = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).transpose(2, 1, 0, 3).reshape(-1, 3)   # label a + (N+1)(b + (N+1)c)
    pm = ff.PolyMesh(np.concatenate(owner).astype(np.int32), nei.astype(np.int32), patches, P, offs,
                     np.concatenate(polys).astype(np.int32))
    box = from_poly_mesh(pm)
    box.n, box.order, box.isUnsplit = n, order, isUnsplit

    k = box.counts()
    mo, ml = int(k["owner"].max()), int(k["losort"].max())
    assert mo > 3 and ml > 3, (order, mo, ml)
    assert max(mo, ml) >= (12 if order == "random" else 24), (order, mo, ml)
    if split_boundary:
        assert k["boundary"].max() >= (5 if periodic_x else 6) and k["multiPatchCells"] > 0
    if periodic_x:
        assert k["coupled"].max() >= 4
    return box


def from_poly_mesh(pm):
    """PolyBox of a foamfile.PolyMesh with points and faces (geometry from PolyMesh.fv_geometry)"""
    geo = pm.fv_geometry()
    nI = pm.nInternalFaces
    lo, up = pm.ldu()
    cps = [p.name for p in pm.patches if p.type == "cyclic"]
    patches = []
    for p in pm.patches:
        s = slice(p.startFace, p.startFace + p.nFaces)
        kind = "cyclic" if p.type == "cyclic" else "wall"
        nr = -(cps.index(p.neighbourPatch) + 1) if kind == "cyclic" else -1
        patches.append(BPatch(p.name, pm.owner[s].astype(np.int32), geo["Sf"][s], geo["Cf"][s], kind, nr))
    return PolyBox(pm.nCells, lo, up, geo["C"], geo["V"], geo["Sf"][:nI], geo["Cf"][:nI], geo["weights"], geo["deltaCoeffs"],
                   patches, pm)


# ---- random graph --------------------------------------------------------------------------------------------------------
def graph(n, k, seed, nIsolated=7, nB=None):
    """tests/test_fv_kernels_cpu._Graph with `nIsolated` cells spread in that have no face at all, random geometry and an unsorted
    boundary list with several faces per cell"""
    from test_fv_kernels_cpu import _Graph
    g = _Graph(n, k, seed)
    rng = np.random.default_rng(seed + 1)
    nC = n + nIsolated
    keep = np.sort(rng.choice(nC, n, replace=False)).astype(np.int32)       # monotone: the face order stays upper-triangular
    lower, upper = keep[g.lower], keep[g.upper]
    nF = len(lower)
    nB = nC // 2 if nB is None else nB
    bfc = rng.integers(0, nC, nB).astype(np.int32)
    C = rng.uniform(0, 1, (nC, 3))
    patches = [BPatch("b0", bfc, rng.uniform(-1, 1, (nB, 3)), rng.uniform(0, 1, (nB, 3)))]
    box = PolyBox(nC, lower, upper, C, rng.uniform(0.5, 2, nC), rng.uniform(-1, 1, (nF, 3)), rng.uniform(0, 1, (nF, 3)),
                  rng.uniform(0.2, 0.8, nF), rng.uniform(1, 2, nF), patches)
    k_ = box.counts()
    assert k_["owner"].max() > 3 and k_["losort"].max() > 3
    assert ((k_["owner"] == 0) & (k_["losort"] == 0)).sum() >= nIsolated
    assert k_["boundary"].max() >= 3 and not np.all(np.diff(bfc) >= 0)
    return box


# ---- coefficient builders ------------------------------------------------------------------------------------------------
def velocity(x):
    """a non-solenoidal velocity, periodic in x: fluxes U(Cf).Sf of both signs that do not sum to zero per cell"""
    return np.stack([1.0 + 0.3 * np.sin(2 * np.pi * x[:, 0]), x[:, 1] * x[:, 1] - 0.3, np.sin(np.pi * x[:, 2])], 1)


def rotation(x):
    """solid-body rotation about the z axis through the box centre"""
    return np.stack([-(x[:, 1] - 0.5), x[:, 0] - 0.5, 0.1 * np.ones(len(x))], 1)


def face_flux(U, Sf):
    return (Sf[:, 0] * U[:, 0] + Sf[:, 1] * U[:, 1]) + Sf[:, 2] * U[:, 2]


def addr(orc, box):
    ps, fc, nr, _ = box.coupled_arrays()
    if ps is None:
        return orc.Addr(box.nCells, box.lower, box.upper)
    return orc.Addr(box.nCells, box.lower, box.upper, ps, fc, neighbRank=nr)


def fvm_case(orc, box, nc, seed=3):
    """nc 1: -laplacian(gamma, p) = s with p fixed on the walls (symmetric); nc 3: ddt + div(phi) - laplacian(nu) of a vector with a
    non-solenoidal phi (asymmetric).  Returns (oracle Addr, d, kw): d with the keys of tests/test_oracle_fvm.py's cases, kw the
    coupled coefficients (couInt, couBou) of the cyclic pair, empty without one.  The coupled internal coefficients enter through
    the glue, so d["diag"] holds the internal faces' part only."""
    from oracle import fvm_oracle as fo
    rng = np.random.default_rng(seed)
    n, V = box.nCells, box.volumes()
    a = addr(orc, box)
    nu = 1.0 if nc == 1 else 0.02
    gamma = rng.uniform(0.5, 1.5, box.nFaces) * nu
    lu, ld = (np.asarray(x) for x in orc.laplacian_fill(a, box.deltaCoeffs(), gamma * box.magSf()))
    if nc == 1:
        lower, upper, diag = None, -lu, -ld
    else:
        cl, cu, cd = (np.asarray(x) for x in orc.convection_fill(a, box.weights(), face_flux(velocity(box.face_centres()), box.Sf())))
        lower, upper, diag = cl - lu, cu - lu, (cd - ld) + V * 50.0
    bfc = box.bFaceCells
    value = rng.uniform(-1, 1, (len(bfc), nc))
    ic, bc = fo.fixedValue_laplacian_coeffs(nu * rng.uniform(0.5, 1.5, len(bfc)) * box.bMagSf(), box.bDeltaCoeffs(), value)
    source = rng.uniform(-1, 1, (n, nc)) * V[:, None]
    d = dict(diag=diag, upper=upper, lower=lower, source=source[:, 0].copy() if nc == 1 else source, bfc=bfc, ic=-ic, bc=-bc, V=V)
    kw = {}
    ps, fc, nr, partner = box.coupled_arrays()
    if ps is not None:
        cps = box.coupled_patches()
        Sfc, Cfc = np.concatenate([p.Sf for p in cps]), np.concatenate([p.Cf for p in cps])
        magc = np.sqrt((Sfc ** 2).sum(1))
        C = box.cell_centres()
        dist = np.abs((Cfc - C[fc])[:, 0]) + np.abs((Cfc - C[fc])[:, 0])[np.concatenate([np.arange(ps[1], ps[2]), np.arange(ps[0], ps[1])])]
        g = nu * rng.uniform(0.5, 1.5, len(fc)) * magc / dist
        if nc == 1:
            intc, bou = g, g.copy()
        else:
            pphi = face_flux(velocity(Cfc), Sfc)
            intc, bou = 0.5 * pphi + g, -0.5 * pphi + g        # distinct both ways
        kw = dict(couInt=intc, couBou=bou)
    return a, d, kw


def mules_case(box, seed=1, combo="one-zero", scale=1e-3):
    """tests/test_mules_cpu.case on a PolyBox: random fields with saturated cells, fluxes of both signs and exactly zero, central
    (unbounded) face values"""
    bfc = box.bFaceCells
    rng = np.random.default_rng(seed)
    n, nF, nB = box.nCells, box.nFaces, len(bfc)
    d = dict(m=box, bfc=bfc, n=n, nF=nF, nB=nB, rDeltaT=50.0)
    d["V"] = box.volumes() * rng.uniform(0.8, 1.2, n)
    d["psi"] = rng.uniform(0, 1, n)
    d["psi"][: n // 5] = 1.0
    d["psi"][n // 5: n // 3] = 0.0
    d["psi0"] = d["psi"].copy()
    d["psiB"] = rng.uniform(0, 1, nB)
    d["phi"], d["phiB"] = rng.uniform(-1, 1, nF) * scale, rng.uniform(-1, 1, nB) * scale
    d["phiB"][: nB // 3] = 0.0
    d["phi"][::13] = 0.0
    d["phiPsi"] = d["phi"] * (0.5 * (d["psi"][box.lower] + d["psi"][box.upper]))
    d["phiPsiB"] = d["phiB"] * d["psiB"]
    kw = {}
    if "rho" in combo:
        kw.update(rho=rng.uniform(0.9, 1.1, n), rho0=rng.uniform(0.9, 1.1, n))
    if "SpSu" in combo:
        kw.update(Sp=-rng.uniform(0, 1, n), Su=rng.uniform(0, 0.1, n))
    d["kw"] = kw
    return d


def asym_matrix(orc, box, seed=5):
    """the convection-diffusion matrix of the engine tests: convection_fill of a non-solenoidal flux minus laplacian_fill, plus a
    time derivative; (Addr, diag, upper, lower)"""
    a = addr(orc, box)
    rng = np.random.default_rng(seed)
    lu, ld = (np.asarray(x) for x in orc.laplacian_fill(a, box.deltaCoeffs(), 0.05 * rng.uniform(0.5, 1.5, box.nFaces) * box.magSf()))
    cl, cu, cd = (np.asarray(x) for x in orc.convection_fill(a, box.weights(), face_flux(velocity(box.face_centres()), box.Sf())))
    return a, (cd - ld) + box.volumes() * 100.0, cu - lu, cl - lu


def sym_matrix(orc, box, seed=6):
    """-laplacian with one pinned cell: (Addr, diag, upper)"""
    a = addr(orc, box)
    rng = np.random.default_rng(seed)
    lu, ld = (np.asarray(x) for x in orc.laplacian_fill(a, box.deltaCoeffs(), rng.uniform(0.5, 1.5, box.nFaces) * box.magSf()))
    diag = -ld
    diag[0] += diag[0]
    return a, diag, -lu


# ---- independent references (not the oracle) -----------------------------------------------------------------------------
U53 = 2.0 ** -53


def _exact_cell_sums(b, fint, fbnd):
    """per cell, the exact rational sum of the face terms (owner +, neighbour -, boundary +), their sum of magnitudes and the
    number of faces; fint (nFaces, k), fbnd (nB, k) as Fractions-able floats"""
    from fractions import Fraction as Fr
    n, k = b.nCells, len(fint[0])
    S = [[Fr(0)] * k for _ in range(n)]
    mag, cnt = np.zeros((n, k)), np.zeros(n)
    for f in range(b.nFaces):
        o, u = b.lower[f], b.upper[f]
        for j in range(k):
            t = fint[f][j]
            S[o][j] += t
            S[u][j] -= t
            mag[o, j] += abs(float(t))
            mag[u, j] += abs(float(t))
        cnt[o] += 1
        cnt[u] += 1
    for f, c in enumerate(b.bFaceCells):
        for j in range(k):
            S[c][j] += fbnd[f][j]
            mag[c, j] += abs(float(fbnd[f][j]))
        cnt[c] += 1
    return S, mag, cnt


def check_exact_gauss_grad(b, phif, phib, got, a):
    """Gauss gradient of phi = a.x + b given its exact values at the face centres: each cell against sum(Sf phi_f)/V in exact
    rational arithmetic within (k+2) 2^-53 sum|Sf phi_f|/V (k faces), and that exact value against a to 1e-12 (the geometry: closed
    planar cells)"""
    from fractions import Fraction as Fr
    prod = lambda S, p: [[Fr(S[f, j]) * Fr(p[f]) for j in range(3)] for f in range(len(p))]
    S, mag, cnt = _exact_cell_sums(b, prod(b.Sf(), phif), prod(b.bSf, phib))
    V = b.volumes()
    bad = []
    for c in range(b.nCells):
        for j in range(3):
            E = S[c][j] / Fr(V[c])
            if abs(float(Fr(got[c, j]) - E)) > (cnt[c] + 2) * U53 * mag[c, j] / V[c]:
                bad.append((c, j, got[c, j], float(E)))
            assert abs(float(E) - a[j]) <= 1e-12 * np.abs(a).max(), (c, j, float(E), a[j])
    assert not bad, f"{len(bad)} gradient components outside the rounding bound, first {bad[:4]}"


def check_closed_sum(b, U, got):
    """surface integral of U.Sf for a constant U (divideByV off): the exact rational sum of the given face terms within
    (k+2) 2^-53 sum|terms|, and that sum itself within the same bound of 0 (closed cells)"""
    from fractions import Fraction as Fr
    fi, fb = b.Sf() @ U, b.bSf @ U
    S, mag, cnt = _exact_cell_sums(b, [[Fr(v)] for v in fi], [[Fr(v)] for v in fb])
    for c in range(b.nCells):
        bound = (cnt[c] + 2) * U53 * mag[c, 0]
        assert abs(float(Fr(got[c]) - S[c][0])) <= bound, (c, got[c], float(S[c][0]))
        assert abs(got[c]) <= 2 * bound, (c, got[c], bound)


def check_interface_normal(b, a, deltaN, nHatf):
    """the exact gradient of a linear alpha: nHatf = a/(|a| + deltaN).Sf within a few ulps per face"""
    n = a / (np.sqrt((a * a).sum()) + deltaN)
    want = face_flux(np.tile(n, (b.nFaces, 1)), b.Sf())
    bound = 8 * U53 * np.abs(b.Sf() * n).sum(1)
    err = np.abs(nHatf - want)
    assert (err <= bound).all(), (int((err > bound).sum()), float((err / np.maximum(bound, 1e-300)).max()))


def check_matrix_products(M, lower, upper, diag, up, low, x, rhs, got):
    """Amul, Tmul and residual of an asymmetric LDU matrix against long-double sums, within (k+2) 2^-53 sum|terms| per row (k
    terms); M: a tests/test_gpu_engine_streams.Mismatches"""
    L_ = np.longdouble
    n = len(diag)
    cnt = 1 + np.bincount(lower, minlength=n) + np.bincount(upper, minlength=n)
    for name, uu, ll in (("Amul", up, low), ("Tmul", low, up)):
        acc = diag.astype(L_) * x.astype(L_)
        mag = np.abs(diag * x)
        np.add.at(acc, lower, uu.astype(L_) * x[upper].astype(L_))
        np.add.at(acc, upper, ll.astype(L_) * x[lower].astype(L_))
        np.add.at(mag, lower, np.abs(uu * x[upper]))
        np.add.at(mag, upper, np.abs(ll * x[lower]))
        bound = (cnt + 2) * U53 * mag
        M.true((np.abs(got[name].astype(L_) - acc) <= bound).all(), f"{name} outside the long-double bound")
        if name == "Amul":
            r = rhs.astype(L_) - acc
            M.true((np.abs(got["residual"].astype(L_) - r) <= (cnt + 3) * U53 * (mag + np.abs(rhs))).all(),
                   "residual outside the long-double bound")


def solenoidal_flux(b):
    """fluxes of U = curl(0, 0, S) with the stream function S = (sin(pi x) sin(pi y))^2/pi through the axis-aligned square faces
    (differences of S at the face's corners, snapped to the point lattice): every closed cell sums to zero up to rounding, and
    S vanishes on the walls, so the boundary flux is 0"""
    S = lambda x, y: (np.sin(np.pi * x) * np.sin(np.pi * y)) ** 2 / np.pi
    N = 2 * b.n
    Sf, Cf = b.Sf(), b.face_centres()
    ax = np.argmax(np.abs(Sf), 1)
    sgn = np.sign(Sf[np.arange(len(Sf)), ax])
    s = np.sqrt(np.abs(Sf[np.arange(len(Sf)), ax]))
    snap = lambda v: np.round(v * N) / N
    x0, x1, y0, y1 = snap(Cf[:, 0] - s / 2), snap(Cf[:, 0] + s / 2), snap(Cf[:, 1] - s / 2), snap(Cf[:, 1] + s / 2)
    cx, cy = snap(Cf[:, 0]), snap(Cf[:, 1])
    phix = sgn * s * (S(cx, y1) - S(cx, y0))
    phiy = -sgn * s * (S(x1, cy) - S(x0, cy))
    return np.where(ax == 0, phix, np.where(ax == 1, phiy, 0.0))


def check_mules_rotation(b, step, nSteps=20):
    """explicit MULES steps of a ball of psi = 1 carried by a discretely solenoidal rotation at Courant 0.25: central face values
    alone over- and undershoot by O(0.05); limited, psi stays within [0, 1] to 1e-12 and sum(V psi) changes only by the boundary flux
    (here 0) to rel 1e-13.  step(psi, phi, phiB, psiB, dt, limited) -> (new psi, limited boundary flux)"""
    V = b.volumes()
    phi = solenoidal_flux(b)
    phiB = np.zeros(len(b.bFaceCells))
    out = np.zeros(b.nCells)
    np.add.at(out, b.lower, np.maximum(phi, 0))
    np.add.at(out, b.upper, np.maximum(-phi, 0))
    dt = 0.25 / (out / V).max()
    C = b.cell_centres()
    psi0 = np.where(((C - np.array([0.5, 0.25, 0.5])) ** 2).sum(1) < 0.15 ** 2, 1.0, 0.0)
    res = {}
    for limited in (False, True):
        psi = psi0.copy()
        mass = (V * psi).sum()
        for _ in range(nSteps):
            new, lpB = step(psi, phi, phiB, psi[b.bFaceCells], dt, limited)
            bflux = dt * lpB.sum()
            assert abs((V * new).sum() - (mass - bflux)) <= 1e-13 * abs(mass), limited
            mass, psi = (V * new).sum(), new
        res[limited] = psi
    assert res[False].min() < -0.05 and res[False].max() > 1.05
    assert res[True].min() >= -1e-12 and res[True].max() <= 1 + 1e-12
