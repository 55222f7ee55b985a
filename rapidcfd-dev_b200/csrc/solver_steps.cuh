// solver_steps.cuh -- device-side scalar logic and the host iteration driver, shared by solvers.cu and gamg.cu
#pragma once
#include "comm.h"
#include "ops.cuh"
#include "solvers.h"

#include <algorithm>

static constexpr double GREAT_ = 1e20;   // SolverPerformance.H:269-275
static constexpr double SMALL_ = 1e-20;
static constexpr double VSMALL_ = 1e-300;

// ---- scalar step: sum partials (fixed order) [+ all-reduce] + scalar logic -------
P2PRed comm_p2p_red(b200ldu_ctx *ctx); // comm.cu

template <int NRED, class G>
int scalar_step_on(Solve &S, double *partials, int nPartials, G g)
{
    b200ldu_ctx *ctx = S.ctx;
    if (ctx->nRanks == 1 || NRED == 0 || ctx->p2p) {
        P2PRed p = (ctx->nRanks > 1 && NRED > 0) ? comm_p2p_red(ctx) : P2PRed();
        scalar_kernel<NRED, true, G><<<1, 256, 0, ctx->stream>>>(partials, nPartials, S.sc, g, p);
        ctx->launches++;
    } else {
        scalar_kernel<NRED, false, G><<<1, 256, 0, ctx->stream>>>(partials, nPartials, S.sc, g, P2PRed());
        ctx->launches++;
        TRY(comm_allreduce_sum(ctx, S.sc->sum, NRED)); // device pointer arithmetic only
        scalar_kernel<0, true, G><<<1, 256, 0, ctx->stream>>>(partials, 0, S.sc, g, P2PRed());
        ctx->launches++;
    }
    KERNEL_CHECK();
    return B200LDU_OK;
}

__device__ __forceinline__ bool check_convergence(SolverScalars *sc)
{
    // SolverPerformance.C:74-85
    bool c = sc->finalResidual < sc->tolerance ||
             (sc->relTol > SMALL_ && sc->finalResidual < sc->relTol * sc->initialResidual);
    sc->converged = c ? 1 : 0;
    return c;
}

__device__ __forceinline__ void hist_put(SolverScalars *sc, double *hist, int i, double v)
{
    if (hist && i < sc->histCap) hist[i] = v;
}

// ---- scalar steps shared by the Krylov solvers ----
// end of an iteration body whose sum|r| is sum[K]: (nIterations++ < maxIter && !converged) || nIterations < minIter
template <int K>
struct EndOfBody {
    double *hist;
    __device__ __forceinline__ void operator()(SolverScalars *sc) const
    {
        sc->finalResidual = sc->sum[K] / sc->normFactor;
        hist_put(sc, hist, sc->nIterations + 1, sc->finalResidual);
        bool conv = check_convergence(sc);
        int n = sc->nIterations;
        sc->nIterations = n + 1;
        bool cont = (n < sc->maxIter && !conv) || (n + 1 < sc->minIter);
        if (!cont) sc->stop = 1;
    }
};
// beta from wArA = sum[0]
struct BetaStep {
    __device__ __forceinline__ void operator()(SolverScalars *s) const
    {
        s->wArAold = s->wArA;
        s->wArA = s->sum[0];
        s->beta = s->wArA / s->wArAold;
    }
};
// alpha from wApA = sum[0], unless the solve is singular (checkSingularity, PCG.C:166-175); false then
struct AlphaStep {
    __device__ __forceinline__ bool operator()(SolverScalars *s) const
    {
        s->wApA = s->sum[0];
        if (!(fabs(s->wApA) / s->normFactor > VSMALL_)) {
            s->singular = 1;
            s->stop = 1;
            return false;
        }
        s->alpha = s->wArA / s->wApA;
        return true;
    }
};

// iteration bodies of a Krylov solve: maxIter + 1 (the last one's judgement always stops), at least minIter
inline long long max_bodies(const b200ldu_controls &c) { return std::max((long long)c.maxIter + 1, (long long)c.minIter); }

#define V2(p) reinterpret_cast<double2 *>(p)
#define CV2(p) reinterpret_cast<const double2 *>(p)

template <int NRED, class G>
int scalar_step(Solve &S, int nPartials, G g)
{
    return scalar_step_on<NRED>(S, S.partials, nPartials, g);
}

// ---------------------------------------------------------------------------
// host driver: enqueue iteration bodies, poll the device stop flag (pipelined)
// ---------------------------------------------------------------------------
template <class Body>
int run_iterations(Solve &S, long long maxBodies, Body body)
{
    b200ldu_ctx *ctx = S.ctx;
    int every = S.c.checkEvery > 0 ? S.c.checkEvery : 8;
    volatile int *flags = (volatile int *)S.pinnedFlags; // two slots
    cudaEvent_t ev[2] = {S.ev[0], S.ev[1]};
    long long enq = 0;
    int chunk = 0;
    bool pending[2] = {false, false};
    cudaGraphExec_t graphExec = nullptr;
    long long launchesPerGraph = 0;
    struct GraphGuard {
        cudaGraphExec_t &g;
        ~GraphGuard()
        {
            if (g) cudaGraphExecDestroy(g);
        }
    } guard{graphExec};
    for (;;) {
        int slot = chunk & 1;
        // before reusing a slot, consume its previous result
        if (pending[slot]) {
            CUDA_TRY(cudaEventSynchronize(ev[slot]));
            pending[slot] = false;
            if (flags[slot]) break;
        }
        if (enq >= maxBodies) {
            // nothing more to enqueue: drain the other slot and leave
            int o = slot ^ 1;
            if (pending[o]) {
                CUDA_TRY(cudaEventSynchronize(ev[o]));
                pending[o] = false;
            }
            break;
        }
        // CUDA graph: after one chunk launched kernel by kernel (attribute set-up, warm caches) a full
        // chunk of `every` bodies (even, so every ping-pong returns to its starting buffers) is captured
        // once and replayed -- the device-side stop flag makes replayed bodies after convergence no-ops.
        const bool fullChunk = (enq + every <= maxBodies) && (every % 2 == 0) && (enq % 2 == 0);
        if (S.useGraph && fullChunk && chunk >= 1) {
            if (!graphExec) {
                long long l0 = ctx->launches;
                cudaGraph_t g = nullptr;
                CUDA_TRY(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed));
                int rcb = B200LDU_OK;
                for (int k = 0; k < every && rcb == B200LDU_OK; k++) rcb = body(enq + k);
                cudaError_t ce = cudaStreamEndCapture(ctx->stream, &g);
                if (rcb != B200LDU_OK) return rcb;
                if (ce != cudaSuccess || !g) {
                    b200_set_error("CUDA graph capture failed: %s", cudaGetErrorString(ce));
                    return B200LDU_ECUDA;
                }
                launchesPerGraph = ctx->launches - l0;
                ctx->launches = l0;
                CUDA_TRY(cudaGraphInstantiate(&graphExec, g, 0));
                cudaGraphDestroy(g);
            }
            CUDA_TRY(cudaGraphLaunch(graphExec, ctx->stream));
            ctx->launches += launchesPerGraph;
            enq += every;
        } else {
            for (int k = 0; k < every && enq < maxBodies; k++, enq++) TRY(body(enq));
        }
        CUDA_TRY(cudaMemcpyAsync((void *)&flags[slot], &S.sc->stop, sizeof(int), cudaMemcpyDeviceToHost,
                                 ctx->stream));
        CUDA_TRY(cudaEventRecord(ev[slot], ctx->stream));
        pending[slot] = true;
        chunk++;
    }
    return B200LDU_OK;
}
