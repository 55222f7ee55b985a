// wallfn_kernels.cuh -- device code of csrc/wallfn.cu: the k-epsilon wall functions.  Kept free of launch syntax and runtime
// calls so that tests/host_kernels/ can compile the same source for the host and run it against oracle/wallfn_oracle.py.
// Reference (WF/ = src/TurbulenceModels/turbulenceModels/RAS/derivedFvPatchFields/wallFunctions/):
//   nutkWallFunction::calcNut   WF/nutWallFunctions/nutkWallFunction/nutkWallFunctionFvPatchScalarField.C:60-130
//   epsilonWallFunction         WF/epsilonWallFunctions/epsilonWallFunction/epsilonWallFunctionFvPatchScalarField.C:
//                               calculate :334-400 (through matrixPatchOperation, lduAddressingFunctors.H:352-400),
//                               calculateTurbulenceFields :231-262, updateCoeffs :540-590
// log, pow and sqrt are the C library's on the host and CUDA's on the device; sqrt rounds correctly on both, log and pow may
// differ in the last bits.
#ifndef B200LDU_WALLFN_KERNELS_CUH
#define B200LDU_WALLFN_KERNELS_CUH
#include <cstddef>

#include "boundary_lists.cuh"

namespace wallfnk
{
namespace // internal linkage: the headers are included by more than one translation unit
{
// nutkWallFunctionFvPatchScalarFieldFunctor per wall face f = faces[i] of the flat boundary list:
// yPlus = Cmu25*y*sqrt(k)/nuw; nut = nuw*(yPlus*kappa/log(E*yPlus) - 1) above yPlusLam, 0 below
__global__ void nutk_kernel(int nW, const int *__restrict__ faces, const int *__restrict__ faceCells, const double *__restrict__ y,
                            const double *__restrict__ k, double nuw, double yPlusLam, double Cmu25, double kappa, double E,
                            double *__restrict__ nutB)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nW) return;
    const int f = faces[i];
    const double yPlus = __ddiv_rn(__dmul_rn(__dmul_rn(Cmu25, y[f]), sqrt(k[faceCells[f]])), nuw);
    nutB[f] = yPlus > yPlusLam ? __dmul_rn(nuw, __dsub_rn(__ddiv_rn(__dmul_rn(yPlus, kappa), log(__dmul_rn(E, yPlus))), 1.0)) : 0.0;
}

// epsilonWallFunction::updateCoeffs of every epsilon-wall patch, per cell: epsilon0 = sum w*Cmu75*pow(k, 1.5)/(kappa*y) and
// G0 = sum w*(nutw + nuw)*mag(snGrad(Uw))*Cmu25*sqrt(k)/(kappa*y) over the cell's wall faces in patch order, faces ascending
// (what matrixPatchOperation sums, starting from 0); then G = G0 and epsilon = epsilon0 in the cell, and epsilon0 becomes
// the patch value of its wall faces.  cw: the corner weight of each boundary face, 0 on faces that are no epsilon wall.
// snGrad of the fixedValue U patch: deltaCoeffs*(Uw - U[cell]) (fvPatchField::snGrad), its magnitude sqrt((x*x + y*y) + z*z).
__global__ void epsilon_wall_kernel(int nCells, fvmk::BoundaryLists L, const double *__restrict__ cw, const double *__restrict__ y,
                                    const double *__restrict__ k, const double *__restrict__ U, const double *__restrict__ Ub,
                                    const double *__restrict__ bDelta, const double *__restrict__ nutB, double nu, double Cmu25,
                                    double Cmu75, double kappa, double *__restrict__ G, double *__restrict__ epsilon,
                                    double *__restrict__ epsB)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nCells || !L.bStart) return;
    const int j0 = L.bStart[c], j1 = L.bStart[c + 1];
    double e0 = 0.0, g0 = 0.0;
    bool wall = false;
    for (int j = j0; j < j1; j++) {
        const int bf = L.bFaces[j];
        const double w = cw[bf];
        if (!(w > 0.0)) continue;
        const double kc = k[c], d = __dmul_rn(kappa, y[bf]), dl = bDelta[bf];
        wall = true;
        double g[3];
#pragma unroll
        for (int q = 0; q < 3; q++) g[q] = __dmul_rn(dl, __dsub_rn(Ub[(size_t)bf * 3 + q], U[(size_t)c * 3 + q]));
        const double mg = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(g[0], g[0]), __dmul_rn(g[1], g[1])), __dmul_rn(g[2], g[2])));
        e0 = __dadd_rn(e0, __ddiv_rn(__dmul_rn(__dmul_rn(w, Cmu75), pow(kc, 1.5)), d));
        const double a = __dmul_rn(__dmul_rn(__dmul_rn(w, __dadd_rn(nutB[bf], nu)), mg), Cmu25);
        g0 = __dadd_rn(g0, __ddiv_rn(__dmul_rn(a, sqrt(kc)), d));
    }
    if (!wall) return;
    G[c] = g0;
    epsilon[c] = e0;
    for (int j = j0; j < j1; j++) {
        const int bf = L.bFaces[j];
        if (cw[bf] > 0.0) epsB[bf] = e0;
    }
}
} // namespace
} // namespace wallfnk
#endif
