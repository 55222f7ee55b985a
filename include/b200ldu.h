/*
 * b200ldu.h -- C ABI of the Hopper-native (sm_90a) lduMatrix linear-solver core.
 *
 * Drop-in boundary for the RapidCFD-dev (OpenFOAM-2.3.x) hot path: a reference-side
 * lduMatrix::solver / preconditioner / smoother registered in the run-time selection
 * tables (LDU/lduMatrix/lduMatrix.H:141-185,297-341,438-460) forwards to these entry
 * points; INTEGRATION.md shows the binding.  "LDU/" = src/OpenFOAM/matrices/lduMatrix/,
 * "FV/" = src/finiteVolume/ of the reference tree.
 *
 * Conventions
 *  - scalar = double, label = int32 (reference etc/bashrc:76, label.H:46-67).
 *  - Every pointer named *_d is DEVICE memory on the context's GPU, in the caller's
 *    OpenFOAM ordering (cells 0..nCells-1, faces sorted by owner then neighbour).
 *    Pointers named *_h are HOST memory.  The caller keeps ownership of everything it
 *    passes in; the library owns handles, derived addressing, renumbering permutations,
 *    banded coefficient copies and all workspace (no cudaMalloc inside ldu_solve after
 *    the first call on a handle).
 *  - Face f: owner lower[f] < neighbour upper[f]; upper[f] = A(owner, neighbour),
 *    lower[f] = A(neighbour, owner); lower == NULL means symmetric
 *    (LDU/lduMatrix/lduMatrix.C:328-345).
 *  - Every function returns 0 on success or a negative B200LDU_E* code; nothing throws
 *    across the ABI; b200ldu_last_error() gives the message for the calling thread.
 *  - No CPU fallback: a missing GPU or a CUDA error is an error return, never a silent
 *    host computation.
 */
#ifndef B200LDU_H
#define B200LDU_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200LDU_OK 0
#define B200LDU_EINVAL -1     /* bad argument */
#define B200LDU_ECUDA -2      /* CUDA runtime / launch failure */
#define B200LDU_ENOSOLVER -3  /* unknown solver name (lduMatrixSolver.C:76-84 prints the table) */
#define B200LDU_ENOPRECOND -4 /* unknown preconditioner / smoother name */
#define B200LDU_EMATRIX -5    /* solver not registered for this matrix kind (sym/asym tables) */
#define B200LDU_ELAYOUT -6    /* mesh cannot be banded (more than 65535 columns in one band) */
#define B200LDU_ENCCL -7
#define B200LDU_ENOLEVELS -8  /* GAMG: no coarse levels created (GAMGSolver.C:174-192) */

typedef struct b200ldu_ctx b200ldu_ctx;       /* one per device (+ NCCL communicator) */
typedef struct b200ldu_addr b200ldu_addr;     /* lduAddressing + banded layout */
typedef struct b200ldu_matrix b200ldu_matrix; /* lduMatrix coefficients in banded form */
typedef struct b200ldu_gamg b200ldu_gamg;     /* cached GAMGAgglomeration (MeshObject) */

/* solver controls: LDU/lduMatrix/lduMatrixSolver.C:167-173, smoothSolver.C:80,
 * JacobiSmoother.C:34-36, GAMGSolver.C:67-77,209-249, GAMGAgglomeration.C:96-128 */
typedef struct b200ldu_controls {
    double tolerance; /* 1e-6 */
    double relTol;    /* 0 */
    int maxIter;      /* 1000 */
    int minIter;      /* 0 */
    int nSweeps;      /* smoothSolver: 1 */
    double omega;     /* Jacobi damping 0.9 */
    int bicgstabRefQuirk; /* 1: mirror PBiCGStab.C:263-270 (second update uses yA) */
    int nCellsInCoarsestLevel, mergeLevels;
    int nPreSweeps, preSweepsLevelMultiplier, maxPreSweeps;
    int nPostSweeps, postSweepsLevelMultiplier, maxPostSweeps;
    int nFinestSweeps;
    int interpolateCorrection;
    int scaleCorrection; /* -1 = matrix.symmetric() */
    int directSolveCoarsest;
    int checkEvery; /* host polls the device convergence flag every k iterations (0 = default 8);
                       the iteration count is decided on the device and is exact */
} b200ldu_controls;

/* solverPerformance: src/OpenFOAM/matrices/LduMatrix/LduMatrix/SolverPerformance.H */
typedef struct b200ldu_perf {
    double initialResidual, finalResidual, normFactor;
    int nIterations, converged, singular;
    char solverName[64]; /* preconditionerName + typeName, DIC/DILU printed as AINV */
} b200ldu_perf;

const char *b200ldu_last_error(void);
void b200ldu_controls_default(b200ldu_controls *c);

/* ---- context ---- */
/* Replaces argList's device selection (src/OpenFOAM/global/argList/argList.C:775-831). */
int b200ldu_ctx_create(int device, b200ldu_ctx **out);
int b200ldu_ctx_destroy(b200ldu_ctx *ctx);
/* Replaces Pstream over MPI (src/Pstream/mpi/UPstream.C:64-79): one NCCL communicator
 * per context.  nccl_unique_id_128 is the 128-byte ncclUniqueId created on rank 0 and
 * broadcast by the host program. */
int b200ldu_comm_unique_id(void *out128);
int b200ldu_comm_init(b200ldu_ctx *ctx, const void *nccl_unique_id_128, int rank, int nRanks);
/* data path of the two exchanges: 1 peer-memory kernels over NVLink, 0 NCCL, -1 not applicable (single rank / no
 * coupled patches).  The peer-memory path needs CUDA IPC between all ranks; otherwise every rank falls back to NCCL. */
int b200ldu_comm_info(const b200ldu_ctx *ctx, const b200ldu_addr *a, int *allreduceP2P, int *haloP2P);
/* stream all work of this context is enqueued on (a cudaStream_t); NULL out => legacy stream */
int b200ldu_ctx_set_stream(b200ldu_ctx *ctx, void *cudaStream);
int b200ldu_ctx_sync(b200ldu_ctx *ctx);

/* ---- lduAddressing (LDU/lduAddressing/lduAddressing.H:119-256) ----
 * lower_h/upper_h: HOST int32[nFaces].  Coupled patches (processor / cyclic interfaces,
 * LDU/lduAddressing/lduInterface): patchStart_h[nPatches+1] offsets into faceCells_h,
 * neighbRank_h[nPatches]: for a processor patch the rank owning the other side; for a cyclic
 * patch -(q+1) where q is the partner patch of this same addressing (cyclicLduInterface::
 * neighbPatchID, face i pairs with face i; scalar fields, no transform).  Cyclic patches are
 * served by the Krylov and smooth solvers and all matrix operations; GAMG rejects them.
 * cellCentres_h: optional HOST double[3*nCells] (fvMesh::C()) used only to choose the
 * band renumbering; NULL => graph-distance embedding of the addressing itself.
 * COLLECTIVE once b200ldu_comm_init has run with nRanks > 1: every rank of the communicator
 * must call it in the same order (one all-gather of the patch table and the cell counts),
 * also a rank whose addressing has no processor patch. */
int b200ldu_addr_create(b200ldu_ctx *ctx, int nCells, int nFaces, const int *lower_h,
                        const int *upper_h, int nPatches, const int *patchStart_h,
                        const int *faceCells_h, const int *neighbRank_h,
                        const double *cellCentres_h, b200ldu_addr **out);
int b200ldu_addr_destroy(b200ldu_addr *a);
/* introspection (tests, DESIGN.md numbers) */
int b200ldu_addr_info(const b200ldu_addr *a, long long *nPadRows, long long *nEntries,
                      long long *nHalo, int *bandRows, int *nBands);
/* face stream of symmetric matrices: stored owner slots (padding included), list items, product-buffer doubles
 * of the largest band, and whether symmetric matrices on this addressing use it (1) or the entry stream (0) */
int b200ldu_addr_face_info(const b200ldu_addr *a, long long *nOwnerSlots, long long *nListItems, int *bufDoubles,
                           int *used);
/* the face stream's table of distinct column and product-slot blocks (one per repeated slice or band list): its
 * 32-bit words and its blocks; 0 and 0 where symmetric matrices use the entry stream */
int b200ldu_addr_face_templates(const b200ldu_addr *a, long long *words, int *count);
/* cell renumbering: perm_h[c] = banded row of caller cell c (HOST int32[nCells]) */
int b200ldu_addr_perm(const b200ldu_addr *a, int *perm_h);

/* ---- lduMatrix coefficients (LDU/lduMatrix/lduMatrix.H:78-96, lduMatrix.C:221-471) ----
 * Copies diag/upper/lower (+ interfaceBouCoeffs/interfaceIntCoeffs, flat over coupled
 * patches in patch order): once into the banded coefficient streams (replaces
 * calcSortCoeffs/lowerSort) and once, caller order, into arrays the matrix owns -- faceH, the
 * b200ldu_fvm_* glue and the GAMG coarse-level assembly read those later.  The caller may free
 * or overwrite its arrays as soon as the call returns; changing coefficients (relax,
 * setReference on the caller's diag) takes another b200ldu_matrix_set to reach the matrix,
 * exactly as a non-const lduMatrix::diag()/upper() access invalidates the reference's sorted
 * copies (lduMatrix.C:238,269).  intCoeffs_d == bouCoeffs_d (same pointer) declares A^T's
 * interface coefficients equal to A's. */
int b200ldu_matrix_create(b200ldu_addr *a, b200ldu_matrix **out);
int b200ldu_matrix_set(b200ldu_matrix *m, const double *diag_d, const double *upper_d,
                       const double *lower_d /* NULL => symmetric */,
                       const double *bouCoeffs_d, const double *intCoeffs_d);
int b200ldu_matrix_destroy(b200ldu_matrix *m);

/* lduMatrix::Amul / Tmul (LDU/lduMatrix/lduMatrixATmul.C:183-261, :264-342) incl. the
 * coupled-interface update; sumA (:345-395); residual (:428-496); H
 * (lduMatrixOperations.C:131-155); H1 (lduMatrixATmul.C:533-554); faceH
 * (lduMatrixTemplates.C:108-149).  Caller-order device vectors. */
int b200ldu_amul(b200ldu_matrix *m, const double *psi_d, double *Apsi_d);
int b200ldu_tmul(b200ldu_matrix *m, const double *psi_d, double *Tpsi_d);
int b200ldu_sumA(b200ldu_matrix *m, double *sumA_d);
int b200ldu_residual(b200ldu_matrix *m, const double *psi_d, const double *source_d, double *rA_d);
int b200ldu_H(b200ldu_matrix *m, const double *psi_d, double *Hpsi_d);
int b200ldu_H1(b200ldu_matrix *m, double *H1_d);
int b200ldu_faceH(b200ldu_matrix *m, const double *psi_d, double *faceHpsi_d);
/* preconditioner::precondition / preconditionT (lduMatrix.H:497-520): name in
 * {none, diagonal, AINV, DIC, DILU} with the reference's aliasing
 * (lduMatrixPreconditioner.C:58-61) */
int b200ldu_precondition(b200ldu_matrix *m, const char *name, int transpose, const double *rA_d,
                         double *wA_d);
/* smoother::smooth (lduMatrix.H:406-412): name in {Jacobi, GaussSeidel(alias)} */
int b200ldu_smooth(b200ldu_matrix *m, const char *name, double omega, double *psi_d,
                   const double *source_d, int nSweeps);

/* banded-order views for benchmarking the kernels exactly as the solvers run them:
 * vectors of b200ldu_vec_len() doubles in banded row order (+ halo tail).  amul_banded exchanges the coupled-patch
 * values into the halo tail of psib (doubles [nPad, vec_len)) before the product: only its rows are read-only. */
long long b200ldu_vec_len(const b200ldu_addr *a);
int b200ldu_to_banded(b200ldu_addr *a, const double *x_d, double *xb_d);
int b200ldu_from_banded(b200ldu_addr *a, const double *xb_d, double *x_d);
int b200ldu_amul_banded(b200ldu_matrix *m, const double *psib_d, double *Apsib_d);
/* one banded kernel by name (amul, tmul, amul_dot, ainv, ainv_dot, jacobi, residual, sumA, H):
 * the per-kernel roofline table of bench.py --kernels */
int b200ldu_bench_op(b200ldu_matrix *m, const char *op, double *xb_d, double *yb_d, const double *bb_d);

/* ---- lduMatrix::solver::New(...)->solve(psi, source, cmpt)
 * (LDU/lduMatrix/lduMatrixSolver.C:43-140; lduMatrix.H:253-258) ----
 * solver in {PCG, PBiCG, PBiCGStab, smoothSolver, diagonal, ICCG, BICCG, GAMG};
 * precondOrSmoother: preconditioner name for the Krylov solvers, smoother for
 * smoothSolver/GAMG.  hist_h (HOST, may be NULL) receives the normalised residual after
 * every iteration (hist[0] = initial).  gamg may be NULL unless solver == GAMG. */
int b200ldu_solve(b200ldu_matrix *m, const char *solver, const char *precondOrSmoother,
                  const b200ldu_controls *controls, b200ldu_gamg *gamg, double *psi_d,
                  const double *source_d, b200ldu_perf *perf, double *hist_h, int histCap);
/* same, HOST psi/source through pinned staging (the "e2e" path: H2D + solve + D2H) */
int b200ldu_solve_host(b200ldu_matrix *m, const char *solver, const char *precondOrSmoother,
                       const b200ldu_controls *controls, b200ldu_gamg *gamg, double *psi_h,
                       const double *source_h, b200ldu_perf *perf, double *hist_h, int histCap);
/* number of library kernels launched on this context since creation */
long long b200ldu_launch_count(const b200ldu_ctx *ctx);
/* device memory of the handles created on this context (addressings, matrices, GAMG hierarchies): the bytes they
 * hold now, and the number of device allocations they have made since the context was created.  Either pointer may
 * be NULL.  Unlike cudaMemGetInfo it counts this library's memory only. */
int b200ldu_ctx_device_mem(const b200ldu_ctx *ctx, long long *liveBytes, long long *nAllocs);

/* ---- GAMGAgglomeration (pair agglomeration, cached on the mesh:
 * LDU/solvers/GAMG/GAMGAgglomerations/..., GAMGAgglomeration.C:132-233) ----
 * faceWeights_h: HOST double[nFaces] (faceAreaPairGAMGAgglomeration.C:56-78).
 * forward: in/out pairGAMGAgglomeration::forward_ (static in the reference).
 * a may be a host-only addressing without coupled patches (b200ldu_layout_debug_create): the
 * hierarchy is then built on the host alone, for nlevels / level_size / restrict_addr, without a GPU. */
int b200ldu_gamg_create(b200ldu_addr *a, const double *faceWeights_h, int nCellsInCoarsestLevel,
                        int mergeLevels, int *forward, b200ldu_gamg **out);
int b200ldu_gamg_destroy(b200ldu_gamg *g);
int b200ldu_gamg_nlevels(const b200ldu_gamg *g);
int b200ldu_gamg_level_size(const b200ldu_gamg *g, int lev, int *nCells, int *nFaces);
/* HOST copies of the level maps (parity tests): restrictAddressing of level lev */
int b200ldu_gamg_restrict_addr(const b200ldu_gamg *g, int lev, int *out_h);
/* HOST copies of what coarse level lev (as restrict_addr) holds, for parity tests.  Returns the element count and
 * copies at most cap elements to out_h (which may be NULL), or B200LDU_EINVAL for a bad lev / what.  Waits for the
 * context stream; changes nothing a later solve sees.
 *   OWNER, NEIGHBOUR   int[nCoarseFaces]  coarse addressing, caller order
 *   FACE_RESTRICT      int[nFineFaces]    fine face -> coarse face, or -(coarse cell + 1) where it collapses into one
 *   FACE_FLIP          int[nFineFaces]    1 where the coarse face runs against the fine one (0 for collapsed faces)
 *   DIAG, UPPER, LOWER double             the last solve's coarse coefficients, caller order; LOWER has 0 elements
 *                                         when that matrix was symmetric
 *   BOU, INT           double             its restricted interface coefficients, coarse patch-face order
 *   PERM               int[nCoarse]       the level's banded row of every coarse cell
 *   INV                double[n * N]      coarsest level only: this rank's rows of the inverse of the coarsest
 *                                         matrix as the solve uploaded them -- banded rows, global banded columns
 *   INV_DIMS           int[3]             coarsest level only: {N, this rank's first row, n}
 * The addressing codes (OWNER ... FACE_FLIP) also serve a host-only hierarchy; coefficients need a solve with
 * this handle first, INV and INV_DIMS a solve with directSolveCoarsest. */
enum {
    B200LDU_GAMG_OWNER, B200LDU_GAMG_NEIGHBOUR, B200LDU_GAMG_FACE_RESTRICT, B200LDU_GAMG_FACE_FLIP,
    B200LDU_GAMG_DIAG, B200LDU_GAMG_UPPER, B200LDU_GAMG_LOWER, B200LDU_GAMG_BOU, B200LDU_GAMG_INT,
    B200LDU_GAMG_PERM, B200LDU_GAMG_INV, B200LDU_GAMG_INV_DIMS
};
long long b200ldu_gamg_debug_get(const b200ldu_gamg *g, int lev, int what, void *out_h, long long cap);
/* Trace of a matrix handle's global sums, for tests that run a solve in lockstep with a CPU restatement.
 * b200ldu_matrix_debug_trace(m, cap) arms it for the handle's later solves (cap records; 0 disarms it).  Every scalar
 * step of a solve then stores one record, in step order: what it summed and the per-CTA partials it summed them from.
 * Unarmed, a solve does exactly what it does without this entry point.  b200ldu_matrix_debug_get(m, what, out_h, cap)
 * copies up to cap doubles of the last solve's trace to out_h and returns how many there are; it waits for the
 * context's stream and changes nothing:
 *   TRACE_RECORDS   double[nRec * 16]  per record: kind (B200LDU_STEP_*), NRED, nPartials, nIterations before the
 *                                      step, sum[0..7] (sum[k], k < NRED, as the step's logic saw it), 4 unused
 *   TRACE_PARTIALS  double[nRec * P]   per record: partials[p * NRED + k], p < nPartials (P: the return value / nRec)
 *   TRACE_SCALARS   double[12]         wArA, wApA, alpha, beta, omega, rA0rA, tAtA, tAsA, normFactor, bodies,
 *                                      psiBodies, and the number of steps the solve ran (more than cap: records lost)
 * nRec = min(steps, cap). */
enum { B200LDU_TRACE_RECORDS, B200LDU_TRACE_PARTIALS, B200LDU_TRACE_SCALARS };
enum {
    B200LDU_STEP_OTHER,     /* a step without a name (GAMG) */
    B200LDU_STEP_INIT,      /* sum|b - A psi|, sum psi */
    B200LDU_STEP_NORM,      /* normFactor */
    B200LDU_STEP_BETA,      /* PCG <w,r> / PBiCG <wA,rT> (operation list) */
    B200LDU_STEP_ALPHA,     /* PCG <Ap,p> / PBiCG <A pA,pT> (operation list) */
    B200LDU_STEP_END,       /* sum|r| closing an iteration (operation list, PBiCGStab, smoothSolver) */
    B200LDU_STEP_PCG_A,     /* fused PCG sweep A: <z,r>, sum|r| of the previous body */
    B200LDU_STEP_PCG_B,     /* fused PCG sweep B: <Ap,p> */
    B200LDU_STEP_PCG_CLOSE, /* fused PCG close: sum|r| of the last body */
    B200LDU_STEP_RHO,       /* PBiCGStab <rA0,rA> */
    B200LDU_STEP_RA0AYA,    /* PBiCGStab <rA0,AyA> */
    B200LDU_STEP_SMAG,      /* PBiCGStab sum|sA| */
    B200LDU_STEP_OMEGA      /* PBiCGStab <tA,tA>, <tA,sA> */
};
int b200ldu_matrix_debug_trace(b200ldu_matrix *m, int cap);
long long b200ldu_matrix_debug_get(const b200ldu_matrix *m, int what, double *out_h, long long cap);
/* The host inverse a GAMG solve uploads for its coarsest level (partial-pivot Gauss-Jordan), on its own: inv_h = A_h^-1,
 * both HOST row-major N x N.  Returns the number of row swaps, or B200LDU_EINVAL for a singular A_h.  No GPU. */
int b200ldu_gamg_debug_invert(int N, const double *A_h, double *inv_h);

/* ---- finiteVolume face-sum loops (caller-order device fields) ----
 * nComp = 1 or 3, AoS.  Boundary faces of all patches concatenated in patch order.
 * fvc::surfaceIntegrate / surfaceSum: FV/finiteVolume/fvc/fvcSurfaceIntegrate.C:138-203,
 * :264-360 ; gaussGrad::gradf: FV/finiteVolume/gradSchemes/gaussGrad/gaussGrad.C:143-242 ;
 * fvmLaplacianUncorrected fill: gaussLaplacianScheme.C:63-64 ; fvmDiv fill:
 * gaussConvectionScheme.C:95-97 ; linear interpolate: surfaceInterpolationScheme.C:272-351 ;
 * addBoundaryDiag/Source: FV/fvMatrices/fvMatrix/fvMatrix.C:209-226,290-312. */
int b200ldu_fv_boundary_set(b200ldu_addr *a, int nBFaces, const int *bFaceCells_h);
int b200ldu_fv_surface_integrate(b200ldu_addr *a, int nComp, const double *ssf_d,
                                 const double *bssf_d, const double *V_d, double *out_d,
                                 int divideByV, int neiSign);
int b200ldu_fv_gauss_grad(b200ldu_addr *a, int nComp, const double *Sf_d, const double *ssf_d,
                          const double *bSf_d, const double *bssf_d, const double *V_d,
                          double *out_d);
int b200ldu_fv_laplacian_fill(b200ldu_addr *a, const double *deltaCoeffs_d,
                              const double *gammaMagSf_d, double *upper_d, double *diag_d);
int b200ldu_fv_convection_fill(b200ldu_addr *a, const double *weights_d, const double *phi_d,
                               double *lower_d, double *upper_d, double *diag_d);
int b200ldu_fv_interpolate_linear(b200ldu_addr *a, int nComp, const double *w_d,
                                  const double *vf_d, double *sf_d);
/* SURVEY.md 8(f) rank 1: linear surface interpolation fused into the face sums (no F-sized
 * temporary).  grad_linear == gauss_grad(interpolate_linear(w, vf)) bit for bit, with bvf the
 * boundary-face values of vf (gaussGrad::calcGrad, gaussGrad.C:256-271); flux_linear is
 * phi = interpolate(U) & Sf per internal face (icoFoam.C:73-78). */
int b200ldu_fv_grad_linear(b200ldu_addr *a, int nComp, const double *Sf_d, const double *w_d,
                           const double *vf_d, const double *bSf_d, const double *bvf_d,
                           const double *V_d, double *out_d);
int b200ldu_fv_flux_linear(b200ldu_addr *a, const double *Sf_d, const double *w_d, const double *U_d,
                           double *phi_d);
int b200ldu_fv_add_boundary_diag(b200ldu_addr *a, const double *internalCoeffs_d, double *diag_d);
int b200ldu_fv_add_boundary_source(b200ldu_addr *a, const double *boundaryCoeffs_d,
                                   double *source_d);

/* ---- fvMatrix glue around the solvers (SURVEY.md section 8 row a17; FV/fvMatrices/fvMatrix/fvMatrix.C,
 * fvScalarMatrix/fvScalarMatrix.C, fvMatrixSolve.C).  The matrix handle supplies diag / upper / lower and, for
 * the coupled patches of its addressing, interfaceIntCoeffs / interfaceBouCoeffs (one scalar per face, used for
 * every component) as given to the last b200ldu_matrix_set.  The non-coupled boundary faces are the flat list of
 * b200ldu_fv_boundary_set (patch order) with internalCoeffs / boundaryCoeffs [nBFaces*nComp]; nComp is 1 or 3,
 * components interleaved.  pnf_d = patchNeighbourField of the coupled patch faces [nCoupledFaces*nComp], which
 * the reference asks of the boundary condition (coupledFvPatchField.H); may be NULL without coupled patches.
 *   add_boundary_diag    diagOut = diagIn + internalCoeffs.component(cmpt)   (fvMatrix.C:209-226); cmpt = -1:
 *                        cmptAv(internalCoeffs) (addCmptAvBoundaryDiag :230-243); diagIn NULL = zero; in place ok
 *   add_boundary_source  sourceOut = sourceIn + boundaryCoeffs [+ interfaceBouCoeffs*pnf when pnf_d != NULL]
 *                        (:290-348, `couples` = pnf_d != NULL)
 *   A                    (diag + cmptAv boundary diagonal)/V                  (:1375-1430)
 *   H                    (lduMatrix::H(psi) + source + boundary source)/V     (:1458-1508, fvScalarMatrix.C:252-283;
 *                        like the reference, without the boundary-diagonal term of stock OpenFOAM)
 *   flux                 internal faces upper*psi[nei] - lower*psi[own]; boundary faces internalCoeffs*psi[cell] -
 *                        boundaryCoeffs (coupled: - interfaceBouCoeffs*pnf)    (:1591-1660)
 *   residual             scalar fields: fvScalarMatrix.C:195-240 as written (coupled neighbour term counted by both
 *                        lduMatrix::residual and addBoundarySource)
 *   relax                in place on diag_d / source_d                         (:1088-1345)
 *   set_reference        source[celli] += diag[celli]*value; diag[celli] *= 2; celli < 0: no-op   (:965-983)
 *   solve                solveSegregated: scalar fvScalarMatrix.C:142-192, vector component loop
 *                        fvMatrixSolve.C:104-226; perf[nComp]; only the banded diagonal is refilled with the folded
 *                        diagonal for the solve and with the matrix's own afterwards (saveDiag): the
 *                        off-diagonal streams are not touched */
/* patchNeighbourField of all coupled patch faces of a caller-order field (coupledFvPatchField::patchNeighbourField:
 * processorFvPatchField.C:196-262 exchange with the neighbour rank, cyclicFvPatchField.C:133-160 partner patch);
 * pnf_d [nCoupledFaces*nComp] in the order of b200ldu_addr_create's faceCells */
int b200ldu_fv_patch_neighbour_field(b200ldu_addr *a, int nComp, const double *field_d, double *pnf_d);
int b200ldu_fvm_add_boundary_diag(b200ldu_matrix *m, int nComp, int cmpt, const double *internalCoeffs_d,
                                  const double *diagIn_d, double *diagOut_d);
int b200ldu_fvm_add_boundary_source(b200ldu_matrix *m, int nComp, const double *boundaryCoeffs_d,
                                    const double *pnf_d, const double *sourceIn_d, double *sourceOut_d);
int b200ldu_fvm_A(b200ldu_matrix *m, int nComp, const double *internalCoeffs_d, const double *V_d, double *A_d);
int b200ldu_fvm_H(b200ldu_matrix *m, int nComp, const double *psi_d, const double *source_d,
                  const double *boundaryCoeffs_d, const double *pnf_d, const double *V_d, double *H_d);
int b200ldu_fvm_flux(b200ldu_matrix *m, int nComp, const double *psi_d, const double *internalCoeffs_d,
                     const double *boundaryCoeffs_d, const double *pnf_d, double *flux_d, double *boundaryFlux_d,
                     double *coupledFlux_d);
int b200ldu_fvm_residual(b200ldu_matrix *m, const double *psi_d, const double *source_d,
                         const double *internalCoeffs_d, const double *boundaryCoeffs_d, const double *pnf_d,
                         double *residual_d);
int b200ldu_fvm_relax(b200ldu_matrix *m, int nComp, double alpha, const double *psi_d,
                      const double *internalCoeffs_d, double *diag_d, double *source_d);
int b200ldu_fvm_set_reference(b200ldu_matrix *m, int celli, int nComp, const double *value_h, double *diag_d,
                              double *source_d);
/* fvMatrix<scalar>::setValues(cells, values) (FV/fvMatrices/fvMatrix/fvMatrix.C:940-950 -> setValuesFromList :456-657, functors
 * :350-450), in place on caller-order arrays, with the boundary faces of b200ldu_fv_boundary_set; single domain only (an
 * addressing with coupled patches is B200LDU_EINVAL).  As the reference's device code writes it, which differs from stock
 * OpenFOAM (DESIGN.md section 2):
 *   psi[cells] = values; source[cells] = values*diag[cells];
 *   every UNSET cell subtracts, owner faces first, then neighbour faces in losort order, lower[f]*value[nei] where the neighbour
 *   is set and upper[f]*value[own] where the owner is set -- the other row's coefficient -- and keeps those couplings;
 *   upper[f] = 0 where the owner is set, lower[f] = 0 where the neighbour is set;
 *   internalCoeffs = boundaryCoeffs = 0 on the boundary faces of set cells.
 * The reference asks a symmetric matrix for its non-const lower(), which makes it asymmetric with a copy of upper
 * (lduMatrix.C:221-238): lower_d is therefore required -- a copy of upper for a symmetric matrix -- and the result is asymmetric.
 * diag is read, not changed.  A cell listed twice must carry equal values: the reference scatters them in no defined order. */
int b200ldu_fvm_set_values(b200ldu_matrix *m, int nSet, const int *cells_d, const double *values_d, double *psi_d,
                           const double *diag_d, double *upper_d, double *lower_d, double *source_d, double *internalCoeffs_d,
                           double *boundaryCoeffs_d);
int b200ldu_fvm_solve(b200ldu_matrix *m, int nComp, const char *solver, const char *precondOrSmoother,
                      const b200ldu_controls *controls, b200ldu_gamg *gamg, double *psi_d, const double *source_d,
                      const double *internalCoeffs_d, const double *boundaryCoeffs_d, const double *pnf_d,
                      b200ldu_perf *perf);

/* ---- k-epsilon wall functions (csrc/wallfn.cu; single domain, boundary faces of b200ldu_fv_boundary_set) ----
 * b200ldu_wallfn_nutk: nutkWallFunction::calcNut (WF/nutWallFunctions/nutkWallFunction/nutkWallFunctionFvPatchScalarField.C:60-130,
 * WF/ = src/TurbulenceModels/turbulenceModels/RAS/derivedFvPatchFields/wallFunctions/) on the nW boundary faces faces_d[]:
 * yPlus = Cmu25*y*sqrt(k[cell])/nuw, nutB[f] = nuw*(yPlus*kappa/log(E*yPlus) - 1) if yPlus > yPlusLam, else 0.  y_d, nutB_d:
 * [nBFaces]; yPlusLam (nutWallFunctionFvPatchScalarField.C:154-168) and Cmu25 = sqrt(sqrt(Cmu)) come from the host.
 * b200ldu_wallfn_epsilon: epsilonWallFunction::updateCoeffs over all epsilon-wall patches (epsilonWallFunctionFvPatchScalarField.C
 * :231-262, :334-400, :540-590): per wall cell epsilon0 = sum w*Cmu75*pow(k, 1.5)/(kappa*y) and G0 = sum w*(nutB + nu)*
 * mag(deltaCoeffs*(Ub - U[cell]))*Cmu25*sqrt(k)/(kappa*y) over its wall faces (patch order, faces ascending, from 0), then
 * G = G0, epsilon = epsilon0 in the cell and epsB = epsilon0 on its wall faces, in place.  cornerWeights_d [nBFaces]: 1/(the
 * number of epsilon-wall faces of the face's cell), 0 on faces of other patches; U_d [nCells*3], Ub_d [nBFaces*3]. */
int b200ldu_wallfn_nutk(b200ldu_addr *a, int nW, const int *faces_d, const double *y_d, const double *k_d, double nuw,
                        double yPlusLam, double Cmu25, double kappa, double E, double *nutB_d);
int b200ldu_wallfn_epsilon(b200ldu_addr *a, const double *cornerWeights_d, const double *y_d, const double *k_d, const double *U_d,
                           const double *Ub_d, const double *bDelta_d, const double *nutB_d, double nu, double Cmu25, double Cmu75,
                           double kappa, double *G_d, double *epsilon_d, double *epsB_d);

/* ---- element-wise field operators between the kernels (SURVEY.md section 8(f) rank 2; the gpuField operator set of
 * src/OpenFOAM/fields/Fields/gpuField/gpuFieldFunctionsM.C:200-330): one rounding per element and operator, so a
 * caller that composes them in the reference's order reproduces the reference's field expressions.  n = elements;
 * a 1-component operand combines with a 3-component one component-wise (scalargpuField * vectorgpuField).
 *   binary op: 0 a+b, 1 a-b, 2 a*b, 3 a/b, 4 min(a,b), 5 max(a,b)
 *   unary  op (n = number of doubles): 0 -a, 1 |a|, 2 s*a, 3 s/a, 4 a+s, 5 s-a, 6 min(a,s), 7 max(a,s), 8 a-s, 9 a/s, 10 a,
 *     11 pos(a) (1 where a >= 0, else 0)
 *   dot3: (a.x*b.x + a.y*b.y) + a.z*b.z per element;  gather: patchInternalField, out[i] = field[cells[i]]
 *   With n = 0 the arrays may be NULL (an empty field hands out no pointer). */
int b200ldu_field_binary(b200ldu_ctx *ctx, int op, long long n, int nCompA, const double *a_d, int nCompB,
                         const double *b_d, double *out_d);
int b200ldu_field_unary(b200ldu_ctx *ctx, int op, long long n, double s, const double *a_d, double *out_d);
int b200ldu_field_dot3(b200ldu_ctx *ctx, long long n, const double *a_d, const double *b_d, double *out_d);
/* magSqr(symm(T)) per element of a tensor field [n*9] (TensorI.H:483-491, SymmTensorI.H:276-284): the k-epsilon production term
 * G = nut*2*magSqr(symm(fvc::grad(U))) (kEpsilon.C:235) takes its tensor from b200ldu_fv_grad_linear(nComp = 3) */
int b200ldu_field_symm_magsqr(b200ldu_ctx *ctx, long long n, const double *tensor_d, double *out_d);
int b200ldu_field_gather(b200ldu_ctx *ctx, int n, int nComp, const int *cells_d, const double *field_d, double *out_d);
/* snGradScheme::snGrad on the internal faces (FV/finiteVolume/snGradSchemes/snGradScheme/snGradScheme.C:101-160):
 * out[f] = deltaCoeffs[f]*(vf[nei] - vf[own]).  With it fvc::laplacian (gaussLaplacianSchemes.C:95-112: div(gamma*snGrad*magSf))
 * and the non-orthogonal correction (correctedSnGrad.C:44-75, gaussLaplacianScheme.C:92-130: corrVecs & interpolate(grad))
 * are compositions of entry points of this header (rapidcfd-dev_b200/fvc.py: laplacian, snGrad_correction). */
int b200ldu_fv_sngrad(b200ldu_addr *a, int nComp, const double *deltaCoeffs_d, const double *vf_d, double *out_d);
/* ---- MULES (FV/fvMatrices/solvers/MULES/MULESTemplates.C) ----
 * b200ldu_mules_limiter = MULES::limiter (:381-745): face limiters lambda (internal faces) / lambdaB (the non-coupled boundary
 * faces of b200ldu_fv_boundary_set) of the anti-diffusive flux phiCorr = phiPsi - phiBD, nLimiterIter sweeps, such that the
 * explicit update keeps psi within [psiMin, psiMax] and the extrema of its face neighbours.  lambda / lambdaB hold the starting
 * limiter on entry (1.0 in MULES::limit).  rho_d / rho0_d NULL = geometricOneField, Sp_d / Su_d NULL = zeroField.  Static mesh.
 * nCoupledFaces: 0, or the number of coupled (processor / cyclic) patch faces of the addressing, which then are the LAST faces of the
 * b200ldu_fv_boundary_set list in the patch order of b200ldu_addr_create; psiB_d holds patchNeighbourField() there (b200ldu_fv_patch_
 * neighbour_field), they are limited by coupledPatchLambdaPfMULESFunctor and after every sweep take the minimum with the other side's
 * limiter (syncTools::syncFaceList, :743; collective over the ranks).  MULES::limit (:748-813) and MULES::explicitSolve (:36-78) are compositions (rapidcfd-dev_b200/mules.py). */
int b200ldu_mules_limiter(b200ldu_addr *a, int nLimiterIter, double rDeltaT, const double *rho_d, const double *rho0_d,
                          const double *psi_d, const double *psi0_d, const double *psiB_d, const double *phiBD_d,
                          const double *phiBDB_d, const double *phiCorr_d, const double *phiCorrB_d, const double *Sp_d,
                          const double *Su_d, const double *V_d, double psiMax, double psiMin, double *lambda_d,
                          double *lambdaB_d, int nCoupledFaces);
/* b200ldu_mules_limiter_corr = MULES::limiterCorr (CMULESTemplates.C:375-704): the limiter of a flux correction phiCorr applied to an
 * already bounded psi (MULES::correct, :35-75; MULES::limitCorr, :706-761: phiCorr *= lambda -- compositions in rapidcfd-dev_b200/
 * mules.py).  phiB_d: the boundary values of the total flux phi (outflow test of the non-coupled faces); extremaCoeff: the solver
 * dictionary's entry (default 0 in the reference).  Everything else as b200ldu_mules_limiter. */
int b200ldu_mules_limiter_corr(b200ldu_addr *a, int nLimiterIter, double rDeltaT, const double *rho_d, const double *psi_d,
                               const double *psiB_d, const double *phiB_d, const double *phiCorr_d, const double *phiCorrB_d,
                               const double *Sp_d, const double *Su_d, const double *V_d, double psiMax, double psiMin,
                               double extremaCoeff, double *lambda_d, double *lambdaB_d, int nCoupledFaces);

/* ---- lduMatrix algebra on caller-order coefficient arrays (LDU/lduMatrix/lduMatrixOperations.C) ----
 * row_sum: mode 0 sumDiag (:36-57), 1 negSumDiag (:59-80), 2 sumMagOffDiag (:83-104); lower_d NULL = symmetric; in place.
 * add_assign: A += B / A -= B with the reference's rules for every combination of diagonal / symmetric / asymmetric
 *   matrices (:235-397); has[3] = {diag, upper, lower} present; hasA is updated (symmetric += asymmetric becomes
 *   asymmetric, diagonal += X takes X's triangles).  scale: A *= cell field (:400-441) or A *= s (sf_d NULL, :444-462). */
int b200ldu_ldu_row_sum(b200ldu_addr *a, int mode, const double *upper_d, const double *lower_d, double *inout_d);
int b200ldu_ldu_add_assign(b200ldu_addr *a, int subtract, double *diagA_d, double *upperA_d, double *lowerA_d, int *hasA,
                           const double *diagB_d, const double *upperB_d, const double *lowerB_d, const int *hasB);
int b200ldu_ldu_scale(b200ldu_addr *a, const double *sf_d, double s, double *diagA_d, double *upperA_d, double *lowerA_d,
                      const int *hasA);

/* ---- limited / upwind interpolation (FV/interpolation/surfaceInterpolation/limitedSchemes/) ----
 * b200ldu_fv_limiter: limiter field on the internal faces, LimitedScheme<..>::calcLimiter (LimitedScheme.C:60-140) with
 *   NVDTVD::r (NVDTVD.H:99-127); scheme "upwind" (0, upwind.H:103-118) | "linear" (1) | "limitedLinear" (coefficient k,
 *   limitedLinear.H:64-101) | "vanLeer" (vanLeer.H:66-85) | "Minmod" (Minmod.H:66-85); scalar field vf, gradc = fvc::grad(vf)
 *   [3 per cell], C = cell centres [3 per cell].
 * b200ldu_fv_limited_weights: w = limiter*cdWeight + (1 - limiter)*pos(faceFlux)
 *   (limitedSurfaceInterpolationScheme.C:155-212); limiter_d NULL => upwind, w = pos(faceFlux) (upwind.H:120-123).
 * The weights feed b200ldu_fv_interpolate_linear / _grad_linear / _flux_linear and b200ldu_fv_convection_fill exactly as the
 * central-differencing weights do (surfaceInterpolationScheme::interpolate(vf, weights), gaussConvectionScheme::fvmDiv). */
int b200ldu_fv_limiter(b200ldu_addr *a, const char *scheme, double k, const double *faceFlux_d, const double *vf_d,
                       const double *gradc_d, const double *C_d, double *limiter_d);
int b200ldu_fv_limited_weights(b200ldu_ctx *ctx, long long n, const double *limiter_d, const double *cdWeights_d,
                               const double *faceFlux_d, double *weights_d);

/* ---- the face passes of the interFoam phase-fraction step (applications/solvers/multiphase/interFoam/alphaEqn.H,
 * src/transportModels/interfaceProperties/interfaceProperties.C; sequenced by rapidcfd-dev_b200/interfoam.py) ----
 * b200ldu_fv_limited_flux: flux_d[f] = outSign*(F*face) with F = fluxSign*faceFlux[f] and face the value of vf that the limited
 *   scheme interpolates under F -- fvc::flux(F, vf, scheme) on the internal faces (gaussConvectionScheme.C:74-84) in one pass:
 *   NVDTVD::r and the limiter as b200ldu_fv_limiter (same scheme names and k), w = lim*cdWeights + (1 - lim)*pos(F)
 *   (limitedSurfaceInterpolationScheme.C:155-212), face = w*(vf[own] - vf[nei]) + vf[nei] (surfaceInterpolationScheme.C:272-351),
 *   every operation rounded on its own: bit for bit b200ldu_fv_limiter -> _limited_weights -> _interpolate_linear ->
 *   b200ldu_field_binary(mul), without their three face fields.  fluxSign, outSign: +1 or -1 (exact), so that
 *   -fvc::flux(-phir, alpha2, scheme) (alphaEqn.H:92-97) is one call.  gradc_d = fvc::grad(vf) [3 per cell] and C_d = cell centres
 *   [3 per cell] may be NULL for "upwind" and "linear".  Boundary faces are the caller's: faceFlux_b*vf_b.
 * b200ldu_vof_interface_flux: interfaceProperties::calculateK up to nHatf (interfaceProperties.C:118-145) and the compression
 *   flux.  Internal faces: gradAlphaf = w*(g[own] - g[nei]) + g[nei] per component of g = gradAlpha_d = fvc::grad(alpha1)
 *   [3 per cell]; nHatfv = gradAlphaf/(mag(gradAlphaf) + deltaN), one division per component (VectorSpaceI.H:621-630), mag =
 *   sqrt((x*x + y*y) + z*z); nHatf_d = (nHatfv.x*Sf.x + nHatfv.y*Sf.y) + nHatfv.z*Sf.z.  With phi_d != NULL also phir_d =
 *   (cAlpha*|phi/magSf|)*nHatf (alphaEqn.H:6, :82); phi_d NULL: magSf_d, phir_d unused.  The non-coupled boundary faces of
 *   b200ldu_fv_boundary_set: the face value of g is the cell value with its normal component replaced by the patch's snGrad,
 *   g += n*(bSnGrad - (n & g)), n = bSf/mag(bSf) (gaussGrad.C:277-303); bSnGrad_d [nBFaces] is 0 for zeroGradient alpha1 and
 *   deltaCoeffs*(alpha_b - alpha_c) for fixedValue; nHatfB_d [nBFaces] from it as on the internal faces.  phic is zero on
 *   non-coupled boundary faces (alphaEqn.H:17-25), so phir has no boundary output.  No contact angles (correctContactAngle).
 *   K = -fvc::div(nHatf) is b200ldu_fv_surface_integrate and a negation. */
int b200ldu_fv_limited_flux(b200ldu_addr *a, const char *scheme, double k, const double *faceFlux_d, const double *vf_d,
                            const double *gradc_d, const double *C_d, const double *cdWeights_d, int fluxSign, int outSign,
                            double *flux_d);
int b200ldu_vof_interface_flux(b200ldu_addr *a, const double *w_d, const double *gradAlpha_d, const double *Sf_d,
                               const double *bSf_d, const double *bSnGrad_d, double deltaN, const double *phi_d,
                               const double *magSf_d, double cAlpha, double *nHatf_d, double *nHatfB_d, double *phir_d);

/* ---- structural self-check of the banded layout (host only, no GPU, no arithmetic);
 * used by the CPU test-suite.  what: 0 perm 1 iperm 2 sliceStart(int64) 3 sliceW(u16)
 * 4 sliceWL(u16) 5 col(u16) 6 code(int32) 7 haloStart 8 haloIdx 9 dims{nPad,nBands,bandRows,
 * nRecv,maxHalo}.  Returns the element count. */
int b200ldu_layout_debug_create(int nCells, int nFaces, const int *lower_h, const int *upper_h,
                                int nPatches, const int *patchStart_h, const int *faceCells_h,
                                const double *cellCentres_h, b200ldu_addr **out);
long long b200ldu_layout_debug_get(const b200ldu_addr *a, int what, void *out, long long cap);
int b200ldu_layout_debug_destroy(b200ldu_addr *a);

#ifdef __cplusplus
}
#endif
#endif
