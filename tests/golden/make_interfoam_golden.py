"""Writes tests/golden/interfoam_golden.npz: the oracle's nHatf, K and phir of a smoothed sphere on 10^3 cells, and alpha1 after two
steps of the phase-fraction step (vanLeer + compression) in its explicit and its MULESCorr branch.  Self-generated: it freezes
oracle/interfoam_oracle.py, so that a later change of the oracle shows.  Run from the repository root:
    python tests/golden/make_interfoam_golden.py"""
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]

import interfoam_cases as ic  # noqa: E402
from oracle import ldu_oracle as orc  # noqa: E402

N = 10


def compute():
    m = importlib.import_module("rapidcfd-dev_b200.mesh").hex_mesh(N)
    a0 = ic.sphere(m)
    o = ic.oracle(orc, m, a0, 1.0)
    phi, _ = ic.rotation_flux(m)
    out = dict(nHatf=o.nHatf, nHatfB=o.nHatfB, K=o.K, phir=(o.cAlpha * np.abs(phi / o.magSf)) * o.nHatf)
    out["alpha_explicit"] = ic.run_oracle(orc, m, a0, ic.controls(nAlphaCorr=2), 2).alpha1
    out["alpha_mulescorr"] = ic.run_oracle(orc, m, a0, ic.controls(MULESCorr=True, nAlphaCorr=2), 2, ic.SOLVER).alpha1
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "interfoam_golden.npz"), **compute())
