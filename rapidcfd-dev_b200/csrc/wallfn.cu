// wallfn.cu -- the k-epsilon wall functions on the device (single domain): nutkWallFunction::calcNut and the epsilon /
// production update of epsilonWallFunction::updateCoeffs.  Kernels and reference lines in wallfn_kernels.cuh; the corner weights
// and yPlusLam are computed once per mesh on the host (rapidcfd-dev_b200/kepsilon.py).
#include "fvmatrix_kernels.cuh"
#include "internal.h"
#include "ldu.h"
#include "wallfn_kernels.cuh"

extern "C" int b200ldu_wallfn_nutk(b200ldu_addr *a, int nW, const int *faces_d, const double *y_d, const double *k_d, double nuw,
                                   double yPlusLam, double Cmu25, double kappa, double E, double *nutB_d)
{
    if (!a || nW < 0 || nW > a->nBFaces || (nW && (!faces_d || !y_d || !k_d || !nutB_d))) return B200LDU_EINVAL;
    CUDA_TRY(cudaSetDevice(a->ctx->device));
    return launch(a->ctx, wallfnk::nutk_kernel, nW, 256, nW, faces_d, a->d_bFaceCells, y_d, k_d, nuw, yPlusLam, Cmu25, kappa, E,
                  nutB_d);
}

extern "C" int b200ldu_wallfn_epsilon(b200ldu_addr *a, const double *cornerWeights_d, const double *y_d, const double *k_d,
                                      const double *U_d, const double *Ub_d, const double *bDelta_d, const double *nutB_d, double nu,
                                      double Cmu25, double Cmu75, double kappa, double *G_d, double *epsilon_d, double *epsB_d)
{
    if (!a || !k_d || !U_d || !G_d || !epsilon_d) return B200LDU_EINVAL;
    if (!a->nBFaces) return B200LDU_OK; // no wall faces
    if (!cornerWeights_d || !y_d || !Ub_d || !bDelta_d || !nutB_d || !epsB_d) return B200LDU_EINVAL;
    if (a->nPatches) {
        b200_set_error("wallfn_epsilon: single domain only (the addressing has %d coupled patches)", a->nPatches);
        return B200LDU_EINVAL;
    }
    CUDA_TRY(cudaSetDevice(a->ctx->device));
    return launch(a->ctx, wallfnk::epsilon_wall_kernel, a->nCells, 128, a->nCells, boundary_lists(a), cornerWeights_d, y_d, k_d, U_d,
                  Ub_d, bDelta_d, nutB_d, nu, Cmu25, Cmu75, kappa, G_d, epsilon_d, epsB_d);
}
