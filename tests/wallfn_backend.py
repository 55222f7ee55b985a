"""The oracle-backed stand-in of tests/oracle_backend.py and tests/interfoam_backend.py with the wall-function entry points of
rapidcfd-dev_b200.capi (fvMatrix::setValues, nutkWallFunction, epsilonWallFunction) over oracle/wallfn_oracle.py, so that the
k-epsilon step with wall functions dry-runs on the CPU.  Test infrastructure only."""
import numpy as np

import interfoam_backend
from oracle import fvm_oracle as fo
from oracle import ldu_oracle as orc
from oracle import wallfn_oracle as wo
from oracle_backend import FieldOps, FvMatrix, _Ctx, _np


class WallFvMatrix(FvMatrix):
    def setValues(self, cells, values, upper, lower):
        """in place on the caller's psi, source, upper, lower, internalCoeffs and boundaryCoeffs (b200ldu_fvm_set_values)"""
        a = self.m.addr
        om = fo.FvMatrix(orc, a.o, 1, _np(self.diag), _np(upper), _np(lower), _np(self.source), _np(self.psi), _np(self.V), a.bfc,
                         _np(self.ic), _np(self.bc))
        wo.set_values(om, _np(cells), _np(values))
        for dst, src in ((self.psi, om.psi), (self.source, om.source), (upper, om.upper), (lower, om.lower), (self.ic, om.ic),
                         (self.bc, om.bc)):
            dst.copy_(FieldOps._t(src))


class Capi(interfoam_backend.Capi):
    FvMatrix = WallFvMatrix

    @staticmethod
    def wallfn_nutk(addr, faces, y, k, nuw, yPlusLam, Cmu25, nutB, kappa=wo.KAPPA, E=wo.E):
        f = _np(faces).astype(np.int64)
        out = _np(nutB).copy()
        out[f] = wo.nutk(_np(y)[f], _np(k)[addr.bfc[f]], nuw, yPlusLam, Cmu25, kappa, E)
        nutB.copy_(FieldOps._t(out))

    @staticmethod
    def wallfn_epsilon(addr, cornerWeights, y, k, U, Ub, bDelta, nutB, nu, Cmu25, Cmu75, G, epsilon, epsB, kappa=wo.KAPPA):
        g, e, eb = wo.epsilon_wall(addr.bfc, _np(cornerWeights), _np(y), _np(k), _np(U), _np(Ub), _np(bDelta), _np(nutB), nu, _np(G),
                                   _np(epsilon), _np(epsB), Cmu25, Cmu75, kappa)
        for dst, src in ((G, g), (epsilon, e), (epsB, eb)):
            dst.copy_(FieldOps._t(src))


def fixture():
    """what the `gpu` fixtures yield: (capi, ctx, torch)"""
    import torch
    return Capi, _Ctx(), torch
