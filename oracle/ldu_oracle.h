/*
 * ldu_oracle.h -- CPU restatement of the RapidCFD-dev lduMatrix hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under rapidcfd-dev_b200/ may include, link or
 * call this.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs use it, and only as the checker or the CPU baseline.
 *
 * PARITY: the reference (SimFlowCFD/RapidCFD-dev @ 975bd36) ships no tests, fixtures or golden
 * vectors for this path (SURVEY.md section 4 / 8c) and cannot be built as a whole in this image
 * (wmake + flex + MPI + all of libOpenFOAM).  Its hot-path SOURCE FILES, however, compile for the
 * host against small type shims (oracle/ref_harness/, `make -C oracle ref` -> oracle/_ref/), and
 * tests/test_reference_functors.py runs them beside this restatement:
 *   PINNED to reference code, bit for bit on hex meshes: the derived addressing arrays
 *     (lduAddressing.C), Amul, Tmul, sumA, residual, H1
 *     (lduMatrixATmul.C), H, faceH (lduMatrixTemplates.C), sumDiag / negSumDiag / sumMagOffDiag, the
 *     coupled-interface update arithmetic (matrixPatchOperation + matrixInterfaceFunctor), AINV
 *     precondition / preconditionT, the Jacobi sweep, smoothSolver, the GAMG V-cycle with scaling and
 *     all sweep controls (GAMGSolverSolve.C, GAMGSolverScale.C), the pair agglomeration maps
 *     (pairGAMGAgglomerate.C), coarse addressing / face restrict / flip maps and combineLevels
 *     (GAMGAgglomerateLduAddressing.C), coarse-matrix assembly (the reference's restriction and
 *     agglomeration functors), the coarsest-level LU (scalarMatrices.C LUDecompose/LUBacksubstitute),
 *     the scalar face sums fvc::surfaceIntegrate / surfaceSum / gaussGrad::gradf (fvcSurfaceIntegrate.C,
 *     gaussGrad.C), the coarse processor interfaces of a decomposed case and their coefficient sums
 *     (GAMGAgglomerateLduAddressing.C interface branch, GAMGInterface.C, processorGAMGInterface.C), the
 *     fvMatrix glue of oracle/fvm_oracle.py for scalar and vector fields (fvMatrix.C, fvMatrixSolve.C,
 *     fvScalarMatrix.C), the finest-level processor exchange + interface update of a decomposed case
 *     (lduMatrixUpdateMatrixInterfaces.C, processorFvPatchScalarField.C, processorGAMGInterfaceField.C) and the
 *     cyclic pairing (cyclicFvPatchField.C), the Laplacian / convection coefficient fills
 *     (gaussLaplacianScheme.C, gaussConvectionScheme.C), the Euler ddt statements of oracle/piso_oracle.py
 *     (EulerDdtScheme.C fvmDdt / fvcDdtPhiCorr, ddtScheme.C fvcDdtPhiCoeff), the linear face interpolation
 *     (surfaceInterpolationScheme.C interpolate(vf)), the matrix sums that form the momentum matrix
 *     (lduMatrixOperations.C operator+= / operator-=; fvMatrix.C operator+ / - / ==);
 *   PINNED to rounding level (the reference's vector updates run unfused on the host, here they are
 *     the FMAs nvcc emits): PCG, PBiCG, PBiCGStab loops incl. iteration counts, names, loop limits
 *     (run-time selection and normFactor -- lduMatrixSolver.C -- bit for bit);
 *   UNPINNED (restated from the source, checked by analytic properties only): the icoFoam
 *     step of oracle/piso_oracle.py as a whole (the order in which it combines the pinned pieces).  Rows with more than three faces per side (coarse GAMG levels,
 *     polyhedral meshes) are summed in plain row order here, the reference unrolls three per side
 *     first: same terms, different association.
 * Analytic checks (dense-matrix SpMV, adjointness, CG exactness on tiny systems, eigenpairs of the
 * 7-point Laplacian, decomposed vs single domain) are in tests/test_oracle_*.py.
 *
 * Conventions: scalar = double, label = int32 (reference: etc/bashrc:76, label.H:46).
 * Face f has owner l[f] < neighbour u[f]; upper[f] = A(l,u), lower[f] = A(u,l);
 * lower == NULL means symmetric (reference lduMatrix.C:328-345).
 *
 * Floating-point contract shared with the CUDA kernels (so SpMV-type results are
 * bit-comparable): products inside a row sum are rounded separately and added in the
 * order  diag, owner-side faces (ascending face), neighbour-side faces (ascending
 * face = losort order), coupled-patch faces (patch order, ascending patch face);
 * the solver AXPYs (x + a*y) are fused multiply-adds, as nvcc contracts them in the
 * reference functors (lduMatrixSolverFunctors.H:7-45).  Compile with
 * -ffp-contract=off; fma() is called explicitly where a contraction is meant.
 */
#ifndef LDU_ORACLE_H
#define LDU_ORACLE_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_addr orc_addr;
typedef struct orc_matrix orc_matrix;

/* Communication hooks.  Serial runs pass NULL.  halo(): given the flat send buffer
 * (psi at patch face cells, all coupled patches concatenated in patch order) fill the
 * flat receive buffer with the neighbour side's values.  sum(): global sum of n
 * doubles in place (rank-ordered sum for reproducibility). */
typedef struct orc_comm {
    void *ctx;
    /* patchStart[nPatches+1] gives the slice of every coupled patch in send/recv (coarse GAMG
     * levels have their own patch sizes; the neighbour ranks are those of the finest level) */
    void (*halo)(void *ctx, const double *send, double *recv, int n, int nPatches, const int *patchStart);
    void (*sum)(void *ctx, double *vals, int n);
    long long nCellsGlobal; /* for gAverage; 0 => local nCells */
    /* all-gather of fixed-size records: every rank contributes n doubles, all[r*n + i] */
    void (*gather)(void *ctx, const double *mine, int n, double *all);
    int rank, nRanks;
} orc_comm;

typedef struct orc_controls {
    double tolerance;   /* default 1e-6  lduMatrixSolver.C:171 */
    double relTol;      /* default 0     lduMatrixSolver.C:172 */
    int maxIter;        /* default 1000  lduMatrixSolver.C:169 */
    int minIter;        /* default 0     lduMatrixSolver.C:170 */
    int nSweeps;        /* smoothSolver, default 1 smoothSolver.C:80 */
    double omega;       /* Jacobi damping, default 0.9 JacobiSmoother.C:34 */
    int bicgstabRefQuirk; /* 1 = mirror PBiCGStab.C:263-270 (psi += omega*yA) */
    /* GAMG keys (GAMGSolver.C:67-77,209-249; GAMGAgglomeration.C:96-98) */
    int nCellsInCoarsestLevel, mergeLevels;
    int nPreSweeps, preSweepsLevelMultiplier, maxPreSweeps;
    int nPostSweeps, postSweepsLevelMultiplier, maxPostSweeps;
    int nFinestSweeps;
    int interpolateCorrection, scaleCorrection /* -1 = matrix.symmetric() */;
    int directSolveCoarsest;
} orc_controls;

typedef struct orc_perf {
    double initialResidual, finalResidual, normFactor;
    int nIterations, converged, singular;
    char solverName[64];
} orc_perf;

void orc_controls_default(orc_controls *c);

/* ---- addressing (lduAddressing.C:169-344) ---- */
orc_addr *orc_addr_create(int nCells, int nFaces, const int *l, const int *u,
                          int nPatches, const int *patchStart, const int *faceCells);
/* neighbour rank of every coupled patch (needed by the multi-rank GAMG agglomeration only) */
void orc_addr_set_neighb_ranks(orc_addr *a, const int *neighbRank);
void orc_addr_free(orc_addr *a);
const int *orc_addr_owner_start(const orc_addr *a);
const int *orc_addr_losort(const orc_addr *a);
const int *orc_addr_losort_start(const orc_addr *a);
const int *orc_addr_lower(const orc_addr *a);
const int *orc_addr_upper(const orc_addr *a);
int orc_addr_npatches(const orc_addr *a);
const int *orc_addr_patch_start(const orc_addr *a); /* nPatches + 1 offsets into faceCells */
const int *orc_addr_face_cells(const orc_addr *a);

void orc_comm_sum(const orc_comm *comm, double *vals, int n); /* global sum of each entry */
/* psi of the cell across every coupled patch face (processor: halo exchange; cyclic: partner patch) */
void orc_patch_neighbour_field(const orc_addr *a, const double *psi, const orc_comm *comm, double *out);

/* ---- matrix ---- */
orc_matrix *orc_matrix_create(const orc_addr *a, const double *diag, const double *upper,
                              const double *lower /* NULL => symmetric */,
                              const double *bouCoeffs, const double *intCoeffs);
void orc_matrix_free(orc_matrix *m);

void orc_amul(const orc_matrix *m, const double *psi, double *Apsi, const orc_comm *comm);
void orc_tmul(const orc_matrix *m, const double *psi, double *Tpsi, const orc_comm *comm);
void orc_sumA(const orc_matrix *m, double *sumA);
void orc_residual(const orc_matrix *m, const double *psi, const double *source, double *rA,
                  const orc_comm *comm);
void orc_H(const orc_matrix *m, const double *psi, double *Hpsi);
void orc_H1(const orc_matrix *m, double *H1);
void orc_faceH(const orc_matrix *m, const double *psi, double *faceHpsi);
void orc_sumDiag(const orc_addr *a, const double *upper, const double *lower, double *diag);
void orc_negSumDiag(const orc_addr *a, const double *upper, const double *lower, double *diag);
void orc_sumMagOffDiag(const orc_addr *a, const double *upper, const double *lower, double *out);

double orc_normFactor(const orc_matrix *m, const double *psi, const double *source,
                      const double *Apsi, double *tmp, const orc_comm *comm);

/* preconditioners: kind 0 none, 1 diagonal, 2 AINV ("DIC"/"DILU" alias to AINV) */
void orc_precondition(const orc_matrix *m, int kind, int transpose, const double *rD,
                      const double *r, double *w);
void orc_jacobi_smooth(const orc_matrix *m, double omega, double *psi, const double *source,
                       int nSweeps, const orc_comm *comm);

/* ---- lockstep with a device solve (tests only; off by default, per thread, single rank) ----
 * An armed reduction hook is called at every global sum of the Krylov solvers, of smoothSolver and of normFactor,
 * after the oracle has formed its own value, and the solve goes on with the value it returns.  site names the
 * call (ORC_SITE_*), iter the iteration body it belongs to (0-based; 0 for the sums before the first body), op the
 * terms: ORC_RED_SUM x[i], ORC_RED_PROD x[i]*y[i] (each product rounded), ORC_RED_MAG |x[i]|.  normFactor hands its
 * 2n terms |Apsi - avg*sumA|, |source - avg*sumA| as x with ORC_RED_MAG.  fn = NULL disarms it. */
enum {
    ORC_SITE_SUMPSI, ORC_SITE_NORMFACTOR, ORC_SITE_SUMMAG0, ORC_SITE_WARA, ORC_SITE_WAPA, ORC_SITE_SUMMAG,
    ORC_SITE_WART, ORC_SITE_WAPT, ORC_SITE_RA0RA, ORC_SITE_RA0AYA, ORC_SITE_SUMMAGS, ORC_SITE_TATA, ORC_SITE_TASA
};
enum { ORC_RED_SUM, ORC_RED_PROD, ORC_RED_MAG };
typedef double (*orc_reduce_fn)(void *ctx, int site, int iter, int op, const double *x, const double *y, int n,
                                double own);
void orc_set_reduce_hook(orc_reduce_fn fn, void *ctx);
/* AINV with the device's association, rD[c]*r[c] formed first and then multiplied by the coefficient (DESIGN.md
 * section 2, exception (i)); 0 (default): the reference's (coeff*rD[c])*r[c].  Per thread. */
void orc_set_staged_ainv(int on);

/* ---- solvers; hist (may be NULL) receives the normalised residual after every
 * iteration body: hist[0] = initial, hist[k] = after k-th body ---- */
int orc_solve(const orc_matrix *m, const char *solver, const char *precondOrSmoother,
              const orc_controls *c, double *psi, const double *source,
              const orc_comm *comm, orc_perf *perf, double *hist, int histCap);

/* ---- GAMG building blocks (exposed for parity tests) ---- */
typedef struct orc_gamg orc_gamg;
orc_gamg *orc_gamg_create(const orc_addr *a, const double *faceWeights /* finest level */,
                          int nCellsInCoarsestLevel, int mergeLevels, int *forwardFlag,
                          const orc_comm *comm /* NULL: single domain */);
void orc_gamg_free(orc_gamg *g);
int orc_gamg_nlevels(const orc_gamg *g);                 /* number of coarse levels */
int orc_gamg_ncells(const orc_gamg *g, int lev);        /* cells of coarse level lev */
int orc_gamg_nfaces(const orc_gamg *g, int lev);
const int *orc_gamg_restrict_addr(const orc_gamg *g, int lev); /* fine(lev)->coarse(lev+1) map; lev 0 = finest */
const int *orc_gamg_face_restrict_addr(const orc_gamg *g, int lev);
const unsigned char *orc_gamg_face_flip(const orc_gamg *g, int lev);
const orc_addr *orc_gamg_addr(const orc_gamg *g, int lev);     /* coarse level addressing */
int orc_gamg_solve(const orc_matrix *m, orc_gamg *g, const char *smoother, const orc_controls *c,
                   double *psi, const double *source, const orc_comm *comm, orc_perf *perf, double *hist,
                   int histCap);
int orc_gamg_npatchfaces(const orc_gamg *g, int lev); /* coupled-patch faces of coarse level lev */
const int *orc_gamg_patch_face_restrict(const orc_gamg *g, int lev); /* fine patch face -> coarse patch face (flat) */
/* GAMGInterface::agglomerateCoeffs over all patches of level lev (GAMGInterface.C:120-172): coarse[cpf] = sum of
 * the fine coefficients mapped to it, in ascending fine patch-face order */
void orc_gamg_agglomerate_patch_coeffs(const orc_gamg *g, int lev, const double *fine, double *coarse);
/* coarse level lev's matrix for the finest matrix m as orc_gamg_solve builds it: diag[nCells], upper/lower[nFaces]
 * (lower written for an asymmetric m only; may be NULL), restricted interface coefficients bou/intc[npatchfaces]
 * (may be NULL) */
void orc_gamg_coarse_matrix(const orc_matrix *m, const orc_gamg *g, int lev, double *diag, double *upper,
                            double *lower, double *bou, double *intc);
/* Opt-in coarsest solve of a given inverse instead of the LU (invRows NULL: back to the LU).  invRows holds this
 * rank's rows of the inverse of the global coarsest matrix, row-major nCells x N, indexed by banded row and by global
 * banded column (rank offset + banded row); perm gives every coarsest cell's banded row.  The correction is
 * x[c] = sum_j inv[perm[c]][j] * b[j], one fused multiply-add per term in ascending j. */
void orc_gamg_set_coarsest_inverse(orc_gamg *g, const double *invRows, const int *perm, int N);
/* descending != 0: the scaling's two sums run from the last cell down (calibrates tolerances for other orders) */
void orc_gamg_set_scale_order(orc_gamg *g, int descending);

/* ---- finite-volume face-sum loops (Appendix A.11) ---- */
void orc_sngrad(const orc_addr *a, int nComp, const double *deltaCoeffs, const double *vf, double *out);
/* nComp = 1 (scalar) or 3 (vector); fields are AoS: x[c*nComp + k]. */
void orc_surface_integrate(const orc_addr *a, int nComp, const double *ssf,
                           int nBFaces, const int *bFaceCells, const double *bssf,
                           const double *V, double *out, int divideByV, int neiSign);
void orc_gauss_grad(const orc_addr *a, int nComp, const double *Sf, const double *ssf,
                    int nBFaces, const int *bFaceCells, const double *bSf, const double *bssf,
                    const double *V, double *out);
void orc_laplacian_fill(const orc_addr *a, const double *deltaCoeffs, const double *gammaMagSf,
                        double *upper, double *diag);
void orc_convection_fill(const orc_addr *a, const double *weights, const double *phi,
                         double *lower, double *upper, double *diag);
void orc_interpolate_linear(const orc_addr *a, int nComp, const double *w, const double *vf, double *sf);
void orc_add_boundary_diag(int nBFaces, const int *bFaceCells, const double *internalCoeffs, double *diag);
void orc_add_boundary_source(int nBFaces, const int *bFaceCells, const double *boundaryCoeffs, double *source);

/* ---- OpenMP all-core variants for the CPU baseline (same numerics, rows in parallel;
 * global sums are per-thread partials combined in thread order) ---- */
int orc_pcg_omp(const orc_matrix *m, int precondKind, const orc_controls *c, double *psi,
                const double *source, orc_perf *perf, int nThreads);
void orc_amul_omp(const orc_matrix *m, const double *psi, double *Apsi, int nThreads);
int orc_max_threads(void);
/* stock OpenFOAM-2.3.x numerics (true DIC, face-loop Amul), serial: CPU baseline only */
int orc_pcg_stock_dic(const orc_matrix *m, const orc_controls *c, double *psi, const double *source,
                      orc_perf *perf);

#ifdef __cplusplus
}
#endif
#endif
