"""Krylov solves in lockstep with the oracle, with the order of the global sums taken out of the comparison.

A solve's only freedom is the order in which it adds the terms of a global sum (DESIGN.md section 2, exception (ii)).
So the oracle is run with each of its global sums replaced by the value the other side computed for the same call
site and iteration (oracle ReduceHook).  Everything else, alpha, beta, omega, the history, the convergence test and
every vector, comes from the oracle's own per-row code and must then match the other side bit for bit.

Each injected sum is checked on its own against the exactly rounded sum S of the oracle's terms at that site and
iteration (once the vectors match bit for bit, those are the other side's terms):  |s - S| <= gamma_d * sum|t_i|,
gamma_d = d u / (1 - d u), u = 2^-53, d the longest chain of roundings a term passes through in the order the code
states (sum_depth).  Without that check a wrong sum would simply be injected and pass unseen.

Vectors that enter only reductions (PBiCG's transposed side, the r of the fused PCG's close) are held only to the
sum bound."""
import math

import numpy as np

U = 2.0 ** -53

# site -> what the oracle sums there (ldu_oracle.h ORC_SITE_*)
SITES = ("sumPsi", "normFactor", "sumMag0", "wArA", "wApA", "sumMag", "wArT", "wApT", "rA0rA", "rA0AyA", "sumMagS",
         "tAtA", "tAsA")


def gamma(d):
    return d * U / (1.0 - d * U)


def sum_depth(nItems, nPartials):
    """Longest rounding chain of one term in a device sum over nItems row pairs (2 rows each) whose per-CTA partials
    (nPartials CTAs of 256 threads) scalar_body adds:
      1   a product the compiler contracts into the sum (nvcc's default -fmad=true) is rounded once less than the
          rounded term it is compared with;
      3   the row pair (and, for normFactor, the two terms of a row) folded before it joins the lane's sum;
      L   the lane's sum over its ceil(nItems / (256 nPartials)) row pairs (a band's lane: slices warp, warp+8, ...;
          an element-wise kernel: its grid-stride loop);
      5   the warp's xor butterfly;  8  block_reduce_store's sum over the block's 8 warps in order;
      P   scalar_body's strided loop over ceil(nPartials / 256) partials;  5 + 8  its 256-thread block reduce."""
    L = max(1, math.ceil(nItems / (256 * nPartials)))
    return 1 + 3 + L + 5 + 8 + max(1, math.ceil(nPartials / 256)) + 5 + 8


def band_depth(nItems, nPartials):
    """the same chain for one CTA's partial (everything before scalar_body)"""
    return 1 + 3 + max(1, math.ceil(nItems / (256 * nPartials))) + 5 + 8


def terms_of(op, x, y):
    """the rounded terms of one oracle sum"""
    if op == "prod":
        return x * y
    if op == "mag":
        return np.abs(x)
    return np.array(x, copy=True)


class Bound:
    """one sum against the exact sum of its terms: ratio = |s - S| / (gamma_d sum|t|) must be <= 1"""

    def __init__(self):
        self.worst = 0.0
        self.where = None
        self.checked = 0

    def ratio(self, s, terms, d):
        S = math.fsum(terms.tolist())
        A = math.fsum(np.abs(terms).tolist())
        self.checked += 1
        if A == 0.0:
            r = 0.0 if s == S else math.inf
        else:
            r = abs(s - S) / (gamma(d) * A)
        return r, S, A

    def check(self, s, terms, d, what, report):
        r, S, A = self.ratio(s, terms, d)
        if r > self.worst:
            self.worst, self.where = r, what
        if not r <= 1.0:
            report.append(f"{what}: sum {s!r} vs exact {S!r} over {len(terms)} terms: |s - S| = {abs(s - S):.3e} "
                          f"> gamma_{d} * sum|t| = {gamma(d) * A:.3e} (ratio {r:.3g})")
        return r


class Report:
    """every failed comparison of a test, so that one failure report names every solver, iteration and field"""

    def __init__(self):
        self.msgs = []

    def append(self, m):
        self.msgs.append(m)

    def bits(self, got, ref, what):
        got, ref = np.asarray(got, np.float64).ravel(), np.asarray(ref, np.float64).ravel()
        if got.shape != ref.shape:
            self.msgs.append(f"{what}: shape {got.shape} != {ref.shape}")
            return False
        bad = np.nonzero(got.view(np.int64) != ref.view(np.int64))[0]
        if len(bad):
            self.msgs.append(f"{what}: {len(bad)} of {len(got)} differ, first at {bad[:4].tolist()}: "
                             f"{got[bad[:4]].tolist()} vs {ref[bad[:4]].tolist()}")
            return False
        return True

    def equal(self, got, ref, what):
        if got != ref:
            self.msgs.append(f"{what}: {got!r} != {ref!r}")
            return False
        return True

    def check(self):
        assert not self.msgs, f"{len(self.msgs)} mismatch(es):\n" + "\n".join(self.msgs)


class OracleRun:
    """One oracle solve with its global sums taken from `sums` ((site, it) -> value; None: its own).  used holds
    the value each site went on with; on_terms(site, it, terms) sees the rounded terms of every sum."""

    def __init__(self, orc, om, solver, pre, psi0, b, sums=None, on_terms=None, staged_ainv=True, **ctl):
        self.used, self.missing = {}, []

        def fn(site, it, op, x, y, own):
            if on_terms is not None:
                on_terms(site, it, terms_of(op, x, y))
            v = own
            if sums is not None:
                v = sums.get((site, it))
                if v is None:
                    self.missing.append((site, it))
                    v = own
            self.used[(site, it)] = v
            return v

        with orc.ReduceHook(fn, staged_ainv=staged_ainv):
            self.psi, self.perf, self.hist = om.solve(solver, pre, psi0, b, **ctl)


# ---- the device's step records -> (site, iteration) ----------------------------------------------------------------
def flavour(solver, fused):
    return {"PCG": "pcgFused" if fused else "pcg", "PBiCG": "pbicg", "PBiCGStab": "pbicgstab",
            "smoothSolver": "smooth"}[solver]


def device_sums(flav, records, kinds):
    """{(site, it): (value, record index, slot)} from a trace's records (LduMatrix.debug_get("records")); kinds
    names the record kinds (LduMatrix.STEP_KINDS)"""
    out = {}
    count = {}
    beta, alpha = {"pcg": ("wArA", "wApA"), "pbicg": ("wArT", "wApT")}.get(flav, (None, None))
    for i, r in enumerate(records):
        kind = kinds[int(r[0])]
        j = count.get(kind, 0)
        count[kind] = j + 1
        put = lambda site, it, k: out.__setitem__((site, it), (float(r[4 + k]), i, k))
        if kind == "init":
            put("sumMag0", 0, 0)
            put("sumPsi", 0, 1)
        elif kind == "norm":
            put("normFactor", 0, 0)
        elif kind == "beta":
            put(beta, j, 0)
        elif kind == "alpha":
            put(alpha, j, 0)
        elif kind == "end":
            put("sumMag", j, 0)
        elif kind == "pcgA":  # sweep A of body j: <z, r_j> and sum|r| after body j-1's update
            put("wArA", j, 0)
            if j > 0:
                put("sumMag", j - 1, 1)
        elif kind == "pcgB":
            put("wApA", j, 0)
        elif kind == "pcgClose":
            put("sumMag", count.get("pcgB", 0) - 1, 1)
        elif kind == "rho":
            put("rA0rA", j, 0)
        elif kind == "rA0AyA":
            put("rA0AyA", j, 0)
        elif kind == "sMag":
            put("sumMagS", j, 0)
        elif kind == "omega":
            put("tAtA", j, 0)
            put("tAsA", j, 1)
    return out


def engine_kinds(flav, pre):
    """record kinds whose partials are one per band (a matrix sweep), by solver and preconditioner"""
    k = {"pcgFused": {"pcgB"}, "pcg": {"alpha"}, "pbicg": {"alpha"}, "pbicgstab": {"rA0AyA", "omega"},
         "smooth": {"end"}}[flav]
    if pre in ("DIC", "DILU", "AINV"):
        k |= {"pcgFused": {"pcgA", "pcgClose"}, "pcg": {"beta"}, "pbicg": {"beta"}}.get(flav, set())
    return k


def expected_scalars(flav, used, last):
    """the scalars a solve that ran bodies 0..last leaves behind, from the sums the oracle used (IEEE divisions in the
    order the device writes them); None where the solve has none"""
    g = used.get
    e = {}
    if flav in ("pcg", "pcgFused", "pbicg"):
        b, a = ("wArT", "wApT") if flav == "pbicg" else ("wArA", "wApA")
        if g((b, last)) is not None and g((a, last)) is not None:
            e["wArA"], e["wApA"] = g((b, last)), g((a, last))
            e["alpha"] = e["wArA"] / e["wApA"]
            e["beta"] = e["wArA"] / (g((b, last - 1)) if last > 0 else 1e20)
    if flav == "pbicgstab" and g(("tAtA", last)) is not None:
        rho, rho0 = g(("rA0rA", last)), g(("rA0rA", last - 1))
        e["rA0rA"], e["tAtA"], e["tAsA"] = rho, g(("tAtA", last)), g(("tAsA", last))
        e["alpha"] = rho / g(("rA0AyA", last))
        e["omega"] = e["tAsA"] / e["tAtA"]
        if last > 0:
            a0 = g(("rA0rA", last - 1)) / g(("rA0AyA", last - 1))
            e["beta"] = (rho / rho0) * (a0 / (g(("tAsA", last - 1)) / g(("tAtA", last - 1))))
    if g(("normFactor", 0)) is not None:
        e["normFactor"] = g(("normFactor", 0)) + 1e-20
    return e
