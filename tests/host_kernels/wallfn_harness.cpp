/*
 * Host execution of the device code of csrc/wallfn.cu (wallfn_kernels.cuh) and of b200ldu_fvm_set_values (fvmatrix_kernels.cuh),
 * in the launch order of the .cu files; built on harness.cpp.  TEST INFRASTRUCTURE ONLY (tests/test_wall_functions_cpu.py).
 */
#include "harness.cpp"

#include <vector>

#include "wallfn_kernels.cuh"

extern "C" {
void hk_set_values(const HostCase *h, int nSet, const int *cells, const double *values, double *psi, const double *diag, double *upper,
                   double *lower, double *source, double *ic, double *bc)
{
    std::vector<int> mask((size_t)h->nCells + 1, 7);
    launch(h->nCells, 256, fvmk::set_values_clear_mask_kernel, h->nCells, mask.data());
    launch(nSet, 256, fvmk::set_values_scatter_kernel, nSet, cells, values, diag, mask.data(), psi, source);
    launch(h->nCells, 128, fvmk::set_values_source_kernel, h->nCells, h->ownerStart, h->u, h->losortStart, h->losort, h->l, upper, lower,
           mask.data(), psi, source);
    launch(h->nFaces, 256, fvmk::set_values_faces_kernel, h->nFaces, h->l, h->u, mask.data(), upper, lower);
    launch(h->nB, 256, fvmk::set_values_boundary_kernel, h->nB, h->bFaceCells, mask.data(), ic, bc);
}

void hk_nutk(int nW, const int *faces, const int *faceCells, const double *y, const double *k, double nuw, double yPlusLam, double Cmu25,
             double kappa, double E, double *nutB)
{
    launch(nW, 256, wallfnk::nutk_kernel, nW, faces, faceCells, y, k, nuw, yPlusLam, Cmu25, kappa, E, nutB);
}

void hk_epsilon_wall(const HostCase *h, const double *cw, const double *y, const double *k, const double *U, const double *Ub,
                     const double *bDelta, const double *nutB, double nu, double Cmu25, double Cmu75, double kappa, double *G,
                     double *epsilon, double *epsB)
{
    const fvmk::BoundaryLists L{h->nB ? h->bStart : nullptr, h->bFaces, nullptr, nullptr};
    launch(h->nCells, 128, wallfnk::epsilon_wall_kernel, h->nCells, L, cw, y, k, U, Ub, bDelta, nutB, nu, Cmu25, Cmu75, kappa, G, epsilon,
           epsB);
}
}
