// solvers.h -- the solve session shared by solvers.cu and gamg.cu
#pragma once
#include "internal.h"

struct SolverScalars;

// Where a solver leaves psi and how its iteration count maps onto the history; the read-back applies these alone.
// The defaults are a Krylov solver's: psi updated in place, one history entry per iteration.
struct SolveResult {
    double *buf[2] = {nullptr, nullptr}; // psi ends in buf[(nIterations * sweepsPerIteration) & 1]
    int sweepsPerIteration = 0;          // Jacobi sweeps that ping-pong psi per counted iteration
    int histEvery = 1;                   // counted iterations per history entry after the first; 0: no history
};

// One solve: the constructor takes the stop-flag pair of its nesting depth, creates two events, decides on CUDA
// graphs, moves to the context's own stream, sizes the device history and uploads the initial scalars (rc: the
// error of that set-up); the destructor undoes all of it on every path.  nIterations0 / converged0 are what a solver
// that runs no scalar step reports.
struct Solve {
    Solve(b200ldu_matrix *m, const b200ldu_controls &c, double *psi, double *src, int histCap, int nIterations0,
          int converged0);
    ~Solve();
    Solve(const Solve &) = delete;
    Solve &operator=(const Solve &) = delete;
    // scalars into perf (one synchronisation), history into hist_h, the banded vector holding psi into *psiOut
    int finish(b200ldu_perf *perf, double *hist_h, double **psiOut);
    // workspace vector k of the matrix (allocated once, reused)
    double *vec(int k) { return k < MAT_NWORK ? banded_vec(m->a, m->mem, MAT_WORK + k) : nullptr; }

    int rc = B200LDU_OK;
    b200ldu_matrix *m;
    b200ldu_ctx *ctx;
    SolverScalars *sc;     // device
    const int *stop;       // &sc->stop: the device's decision to end the solve
    int n2, nBands;        // row pairs of a banded vector; CTAs (and partials) of a matrix sweep
    double *partials;      // device
    double *psi, *src;     // banded device vectors
    b200ldu_controls c;
    double *hist = nullptr; // device
    int histCap; // caller's history capacity, 0 without one
    int *pinnedFlags = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    bool useGraph = false; // replay iteration chunks as a CUDA graph
    SolveResult result;

  private:
    int open(int nIterations0, int converged0);
    bool swapped_ = false; // runs on the context's own stream instead of userStream_
    cudaStream_t userStream_ = nullptr;
    bool entered_ = false; // counted in the nesting depth
};

int init_residual(Solve &S, const double *psi, const double *b, const double *wA, double *rA, double *tmp,
                  const double *wT = nullptr, double *rT = nullptr); // solvers.cu
int solve_banded(b200ldu_matrix *m, const char *solver, const char *pre, const b200ldu_controls *controls,
                 b200ldu_gamg *gamg, double *psi_b, double *src_b, b200ldu_perf *perf, double *hist_h,
                 int histCap, double **resultBuf);
