// ops.cuh -- engine operators (row-gather family) and generic elementwise / scalar
// kernels used by the solvers.  See engine.cuh for the Op concept.
#pragma once
#include "engine.cuh"
#include "ldu.h"

// device-resident solver state: alpha/beta and the convergence decision never leave
// the GPU inside the iteration loop (the reference synchronises the host three times
// per PCG iteration: PCG.C:142,166,195).
struct SolverScalars {
    double sum[8];  // latest (all-reduced) sums
    double wArA, wArAold, wApA, alpha, beta, omega;
    double rA0rA, rA0rAold, tAtA, tAsA;
    double normFactor, initialResidual, finalResidual, average, sumMag0;
    double tolerance, relTol, nCellsGlobal;
    int nIterations, converged, singular, stop;
    int maxIter, minIter, histCap, nSweeps;
    int bodies; // fused PCG: iteration bodies whose A.p product has been formed
    int psiBodies; // fused PCG: bodies whose alpha p has been added to psi (bodies - 1 or bodies)
    // fused PCG, deferred scalar steps (DeferredStep): steps completed (low 32 bits) | stop (bit 63), published by CTA 0 of
    // each sweep with one release store and read by every other CTA with one acquire load.  On its own 128-byte line so
    // that the waiting CTAs' polling does not slow down CTA 0's writes to the scalars above.
    alignas(128) unsigned long long gate;
    unsigned long long gatePad[15];
};

// Page-locked host area of a context (b200ldu_ctx::pinned), allocated once with the context and never moved: a
// nested solve must not free what the outer solve is still polling.
constexpr int SOLVE_MAX_DEPTH = 8; // GAMG nests one Krylov solve; deeper nesting is refused
struct PinnedArea {
    int flags[SOLVE_MAX_DEPTH][2]; // stop-flag pair polled by the solve at each nesting depth (run_iterations)
    SolverScalars scalars;         // read back at the end of a solve
    unsigned long long peerErr;    // a bounded wait on a peer's flag gave up (engine.cuh spin_until)
};

struct OpBase {
    const int *stop = nullptr;
    double *partials = nullptr;
    int waitHalo = 0; // 1: a peer-memory halo exchange of the staged vector is in flight
    // first thing every CTA of an engine kernel does; false => the CTA exits (the device has decided to stop)
    __device__ __forceinline__ bool prologue(const LayoutDev &) const { return !(stop && *stop); }
    // row-sum terms: add(acc, prod(v, a)) = acc + v*a; Residual, OffDiag and CoeffSum replace them
    __device__ __forceinline__ double prod(double v, double a) const { return __dmul_rn(v, a); }
    __device__ __forceinline__ double add(double acc, double p) const { return __dadd_rn(acc, p); }
    __device__ __forceinline__ double identity() const { return -0.0; } // x + -0 == x, also for x = -0
};

// operators that stage the vector x unchanged
struct StageXOp : OpBase {
    static constexpr bool STAGED = true;
    const double *x;
    __device__ __forceinline__ double stage(int g) const { return x[g]; }
    __device__ __forceinline__ double2 stage_own(int r) const
    {
        // returned as two doubles: a returned double2 lvalue is copied as four 32-bit words, which
        // renumbers the registers of the staging loop
        const double2 a = *reinterpret_cast<const double2 *>(x + r);
        return make_double2(a.x, a.y);
    }
};

// ---- Amul / Tmul: out = diag*x + sum v*x[c]  (lduMatrixATmul.C:78-137), with the sums of AmulSum (ldu.h) ----
template <AmulSum MODE>
struct AmulOp : StageXOp {
    static constexpr int NRED = MODE == AMUL_ONLY ? 0 : ((MODE == AMUL_OUT_X || MODE == AMUL_OUT_AUX) ? 1 : 2);
    static constexpr bool LOCAL = false;
    const double *diag, *aux;
    double *out;
    __device__ __forceinline__ double init(int r, double a) const { return __dmul_rn(diag[r], a); }
    __device__ __forceinline__ void finish(int r, double acc0, double acc1, double a0, double a1, double *red) const
    {
        *reinterpret_cast<double2 *>(out + r) = make_double2(acc0, acc1);
        if (MODE == AMUL_OUT_X) red[0] += acc0 * a0 + acc1 * a1;
        if (MODE == AMUL_AUX_X_OUT_X) {
            red[0] += aux[r] * a0 + aux[r + 1] * a1;
            red[1] += acc0 * a0 + acc1 * a1;
        }
        if (MODE == AMUL_OUT_AUX) red[0] += acc0 * aux[r] + acc1 * aux[r + 1];
        if (MODE == AMUL_OUT_OUT_OUT_AUX) {
            red[0] += acc0 * acc0 + acc1 * acc1;
            red[1] += acc0 * aux[r] + acc1 * aux[r + 1];
        }
    }
};

// ---- AINV ("DIC"/"DILU"): w = rD*(r - sum v*(rD[c]*r[c]))  (AINVPreconditionerF.H:42-99)
// The reference evaluates upper[f]*rD[nei]*r[nei] left to right; here the band stages
// t = rD*r once (one shared-memory tile, one gather per halo column and vector) and the
// sweep streams the matrix's own coefficients -- no scaled copy of the matrix, exactly the
// bytes of an Amul, and it works on the shared-coefficient layout.  The association differs
// from the reference's by one rounding per term: parity with the oracle is to ~1e-15
// relative per row, not bit-exact (tests state the tolerance).  Optional fused dot
// <w, dotv> (wArA with dotv = r; wArT with dotv = rT).
template <int NRED_>
struct AinvOp : OpBase {
    static constexpr bool STAGED = true, LOCAL = true;
    static constexpr int NRED = NRED_;
    const double *r, *rD, *dotv;
    double *out;
    __device__ __forceinline__ double stage(int g) const { return __dmul_rn(rD[g], r[g]); }
    __device__ __forceinline__ double2 stage_own(int row) const
    {
        double2 rr = *reinterpret_cast<const double2 *>(r + row);
        double2 dd = *reinterpret_cast<const double2 *>(rD + row);
        return make_double2(__dmul_rn(dd.x, rr.x), __dmul_rn(dd.y, rr.y));
    }
    __device__ __forceinline__ double init(int, double) const { return 0.0; }
    __device__ __forceinline__ void finish(int row, double acc0, double acc1, double, double, double *red) const
    {
        double2 d = *reinterpret_cast<const double2 *>(rD + row);
        double2 rr = *reinterpret_cast<const double2 *>(r + row);
        double w0 = __dmul_rn(d.x, __dsub_rn(rr.x, acc0));
        double w1 = __dmul_rn(d.y, __dsub_rn(rr.y, acc1));
        *reinterpret_cast<double2 *>(out + row) = make_double2(w0, w1);
        if (NRED == 1) {
            double d0 = dotv ? dotv[row] : rr.x, d1 = dotv ? dotv[row + 1] : rr.y;
            red[0] += w0 * d0 + w1 * d1;
        }
    }
};

// ---- Jacobi sweep (JacobiSmootherF.H:51-109; omega-damped, old psi everywhere) ----
struct JacobiOp : StageXOp {
    static constexpr int NRED = 0;
    static constexpr bool LOCAL = false;
    const double *diag, *b;
    double *out;
    double omega;
    __device__ __forceinline__ double init(int, double) const { return 0.0; }
    __device__ __forceinline__ double row(int r, double acc, double a) const
    {
        double rD = __ddiv_rn(1.0, diag[r]);
        double w = __dmul_rn(omega, rD);
        double extra = __dadd_rn(__dmul_rn(1 - omega, a), __dmul_rn(w, b[r]));
        return __dsub_rn(extra, __dmul_rn(w, acc));
    }
    __device__ __forceinline__ void finish(int r, double acc0, double acc1, double a0, double a1, double *) const
    {
        *reinterpret_cast<double2 *>(out + r) = make_double2(row(r, acc0, a0), row(r + 1, acc1, a1));
    }
};

// ---- residual: rA = (b - diag*x) - sum v*x ; fused sum|rA|  (lduMatrixATmul.C:397-496)
template <int NRED_>
struct ResidualOp : StageXOp {
    static constexpr int NRED = NRED_;
    static constexpr bool LOCAL = false;
    const double *diag, *b;
    double *out;
    __device__ __forceinline__ double init(int r, double a) const { return __dsub_rn(b[r], __dmul_rn(diag[r], a)); }
    __device__ __forceinline__ double add(double acc, double p) const { return __dsub_rn(acc, p); }
    __device__ __forceinline__ double identity() const { return 0.0; } // x - +0 == x
    __device__ __forceinline__ void finish(int r, double acc0, double acc1, double, double, double *red) const
    {
        *reinterpret_cast<double2 *>(out + r) = make_double2(acc0, acc1);
        if (NRED == 1) red[0] += fabs(acc0) + fabs(acc1);
    }
};

// ---- coefficient-only row sums: sumA (all entries, + diag), H1 (local, negated) ----
template <bool LOCAL_, bool NEG_>
struct CoeffSumOp : OpBase {
    static constexpr bool STAGED = false, LOCAL = LOCAL_;
    static constexpr int NRED = 0;
    const double *diag; // nullptr => start from 0
    double *out;
    __device__ __forceinline__ double stage(int) const { return 0.0; }
    __device__ __forceinline__ double2 stage_own(int) const { return make_double2(0, 0); }
    __device__ __forceinline__ double init(int r, double) const { return diag ? diag[r] : 0.0; }
    __device__ __forceinline__ double prod(double v, double) const { return v; }
    __device__ __forceinline__ double add(double acc, double p) const { return NEG_ ? __dsub_rn(acc, p) : __dadd_rn(acc, p); }
    __device__ __forceinline__ double identity() const { return NEG_ ? 0.0 : -0.0; }
    __device__ __forceinline__ void finish(int r, double acc0, double acc1, double, double, double *) const
    {
        *reinterpret_cast<double2 *>(out + r) = make_double2(acc0, acc1);
    }
};

// ---- off-diagonal product sums: H = -(sum v*x) local only (lduMatrixOperations.C:107-155);
// GAMG interpolate: psi' = -(sum v*x)/diag over all entries (GAMGSolverInterpolate.C:45-110)
template <bool LOCAL_, bool DIVDIAG_>
struct OffDiagOp : StageXOp {
    static constexpr int NRED = 0;
    static constexpr bool LOCAL = LOCAL_;
    const double *diag;
    double *out;
    __device__ __forceinline__ double init(int, double) const { return 0.0; }
    __device__ __forceinline__ double add(double acc, double p) const { return DIVDIAG_ ? __dadd_rn(acc, p) : __dsub_rn(acc, p); }
    __device__ __forceinline__ double identity() const { return DIVDIAG_ ? -0.0 : 0.0; }
    __device__ __forceinline__ void finish(int r, double acc0, double acc1, double, double, double *) const
    {
        if (DIVDIAG_) {
            acc0 = __ddiv_rn(-acc0, diag[r]);
            acc1 = __ddiv_rn(-acc1, diag[r + 1]);
        }
        *reinterpret_cast<double2 *>(out + r) = make_double2(acc0, acc1);
    }
};

// ---------------------------------------------------------------------------
// elementwise kernels with fused reductions.  f(i2, red) handles elements 2*i2, 2*i2+1
// (vectors are 16-byte aligned and of even length => 128-bit loads/stores).
// ---------------------------------------------------------------------------
constexpr int EW_THREADS = 256;

// prologue of an element-wise kernel that has no deferred scalar step to run
struct NoPrologue {
    __device__ __forceinline__ bool run() const { return true; }
};

// pre.run() first: a deferred scalar step (DeferredStep below) or nothing
template <int NRED, class F, class Pre>
__global__ void __launch_bounds__(EW_THREADS) ew_kernel(int n2, const int *stop, double *partials, F f, Pre pre)
{
    if (stop && *stop) return;
    if (!pre.run()) return;
    double red[NRED > 0 ? NRED : 1];
#pragma unroll
    for (int k = 0; k < (NRED > 0 ? NRED : 1); k++) red[k] = 0;
    for (int i = blockIdx.x * EW_THREADS + threadIdx.x; i < n2; i += gridDim.x * EW_THREADS) f(i, red);
    if (NRED > 0) block_reduce_store<(NRED > 0 ? NRED : 1), EW_THREADS>(red, partials, blockIdx.x);
}

inline int ew_grid(const b200ldu_ctx *ctx, int n2)
{
    int want = (n2 + EW_THREADS - 1) / EW_THREADS;
    int cap = ctx->smCount * 8;
    return want < 1 ? 1 : (want < cap ? want : cap);
}

template <int NRED, class F, class Pre = NoPrologue>
int ew_launch(b200ldu_ctx *ctx, int n2, const int *stop, double *partials, int *nPartialsOut, F f, Pre pre = Pre())
{
    int g = ew_grid(ctx, n2);
    ew_kernel<NRED, F, Pre><<<g, EW_THREADS, 0, ctx->stream>>>(n2, stop, partials, f, pre);
    ctx->launches++;
    if (nPartialsOut) *nPartialsOut = g;
    KERNEL_CHECK();
    return B200LDU_OK;
}

// sums NRED interleaved partial streams in fixed order, then thread 0 runs the scalar
// logic g(sc).  One CTA.  With more than one rank the per-rank sums are combined either
//  * over peer memory (p2p.nRanks > 1): thread 0 stores its sums + a sequence flag into
//    every rank's mailbox (NVLink peer stores), waits until every rank's flag for this
//    sequence number has arrived in its own mailbox and adds the contributions in rank
//    order -- one kernel, no NCCL call, bit-identical result on every rank; or
//  * through ncclAllReduce between a sum-only and a logic-only launch (scalar_step_on).
template <int NRED, bool RUN_LOGIC, class G>
__device__ __forceinline__ void scalar_body(const double *partials, int nPartials, SolverScalars *sc,
                                            G &g, const P2PRed &p2p)
{
    if (NRED > 0) {
        // thread t adds partials t, t+256, ... in that order (fixed => deterministic); the loads of eight of them are
        // issued together, all NRED sums of a partial at once: the step is serial time for the whole GPU
        double red[NRED > 0 ? NRED : 1];
#pragma unroll
        for (int k = 0; k < (NRED > 0 ? NRED : 1); k++) red[k] = 0;
        for (int base = threadIdx.x; base < nPartials; base += 256 * 8) {
            double v[8][NRED > 0 ? NRED : 1];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int i = base + u * 256;
                if (i < nPartials)
#pragma unroll
                    for (int k = 0; k < NRED; k++) v[u][k] = __ldcg(partials + (size_t)i * NRED + k);
            }
#pragma unroll
            for (int u = 0; u < 8; u++)
                if (base + u * 256 < nPartials)
#pragma unroll
                    for (int k = 0; k < NRED; k++) red[k] += v[u][k];
        }
        __shared__ double tot[NRED > 0 ? NRED : 1];
        block_reduce_store<(NRED > 0 ? NRED : 1), 256>(red, tot, 0);
        __syncthreads();
        if (p2p.nRanks > 1) {
            // one thread per peer: the R peer stores, flags and waits proceed concurrently, so the
            // exchange costs one NVLink round trip instead of R
            __shared__ double got[P2P_MAXR][NRED > 0 ? NRED : 1];
            const unsigned long long seq = *p2p.seq + 1;
            const int par = (int)(seq & 1);
            if (threadIdx.x < p2p.nRanks) {
                const int r = threadIdx.x;
                double *dst = p2p.mail[r] + ((size_t)(par * P2P_MAXR + p2p.rank) * 8);
                for (int k = 0; k < NRED; k++) dst[k] = tot[k];
                __threadfence_system();
                unsigned long long *f = p2p.flag[r] + (par * P2P_MAXR + p2p.rank);
                asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(f), "l"(seq) : "memory");
                spin_until(p2p.flag[p2p.rank] + (par * P2P_MAXR + r), seq, p2p.seq + 7);
                const double *src = p2p.mail[p2p.rank] + ((size_t)(par * P2P_MAXR + r) * 8);
                for (int k = 0; k < NRED; k++) got[r][k] = __ldcg(src + k);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                for (int k = 0; k < NRED; k++) {
                    double acc = 0;
                    for (int r = 0; r < p2p.nRanks; r++) acc += got[r][k]; // rank order => same bits everywhere
                    sc->sum[k] = acc;
                }
                *p2p.seq = seq;
            }
        } else if (threadIdx.x == 0) {
            for (int k = 0; k < NRED; k++) sc->sum[k] = tot[k];
        }
    }
    if (RUN_LOGIC && threadIdx.x == 0) g(sc);
}

template <int NRED, bool RUN_LOGIC, class G>
__global__ void __launch_bounds__(256) scalar_kernel(const double *partials, int nPartials,
                                                     SolverScalars *sc, G g, P2PRed p2p)
{
    if (sc->stop) return;
    scalar_body<NRED, RUN_LOGIC>(partials, nPartials, sc, g, p2p);
}

// ---------------------------------------------------------------------------
// Deferred scalar step: the step that closes sweep n (fixed-order sum of its per-band partials, cross-rank
// all-reduce over the peer mailboxes, alpha / beta / convergence logic) runs in the PROLOGUE of sweep n+1's
// kernel instead of a one-CTA launch of its own: CTA 0 does the work (the kernel boundary has made the
// partials visible) and releases a generation counter; every other CTA waits for it before it touches
// anything that depends on the scalars.  Saves two launches and two kernel boundaries per PCG iteration.
// `want` is baked into the launch (graph-replayable): position of this sweep in the chunk of iterations.
// ---------------------------------------------------------------------------
template <int NRED, class G>
struct DeferredStep {
    const double *partials;
    int nPartials;
    SolverScalars *sc;
    G g;
    P2PRed p2p;
    unsigned want, mod; // wait until stepGen % mod == want
    int active;         // 0: nothing to close (first sweep of a solve)
    __device__ __forceinline__ bool run() const
    {
        if (!active) return *reinterpret_cast<volatile const int *>(&sc->stop) == 0;
        __shared__ unsigned long long gateSeen;
        if (blockIdx.x == 0) {
            if (*reinterpret_cast<volatile const int *>(&sc->stop)) {
                // stopped before this sweep (e.g. converged at the initial residual): tell the waiting CTAs
                if (threadIdx.x == 0) {
                    const unsigned long long v = sc->gate | (1ull << 63);
                    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(&sc->gate), "l"(v) : "memory");
                }
                return false;
            }
            G gg = g;
            scalar_body<NRED, true>(partials, nPartials, sc, gg, p2p);
            __syncthreads();
            if (threadIdx.x == 0) {
                const unsigned long long next = ((sc->gate & 0xffffffffull) + 1) | ((unsigned long long)(sc->stop != 0) << 63);
                asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(&sc->gate), "l"(next) : "memory");
                gateSeen = next;
            }
        } else {
            if (threadIdx.x == 0) {
                unsigned long long v, t0 = 0;
                unsigned spins = 0;
                for (;;) {
                    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(&sc->gate) : "memory");
                    // this sweep's step is done, or an earlier sweep already stopped the solve (then nothing advances)
                    if ((unsigned)(v & 0xffffffffull) % mod == want || (v >> 63)) break;
                    __nanosleep(64);
                    if ((++spins & 0x3ffu) == 0) { // bounded: CTA 0 is dispatched first in practice, not by contract
                        unsigned long long now;
                        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
                        if (!t0) t0 = now;
                        if (now - t0 > 20000000000ull) {
                            if (p2p.seq) atomicExch(p2p.seq + 7, 2ull);
                            v |= 1ull << 63;
                            break;
                        }
                    }
                }
                gateSeen = v;
            }
        }
        __syncthreads();
        return (gateSeen >> 63) == 0;
    }
};

// ---- fused PCG kernels (PCG.C:131-205 regrouped into two matrix sweeps per iteration) ----
// K_A: applies the residual update of the PREVIOUS body (r -= alpha w; alpha from the
// device scalars) while staging r, then preconditions: z = rD*(r - sum v*(rD*r)[c]); fused
// sums <z,r> and sum|r|.  r is ping-ponged (other bands read the old halo values).
template <class Pre>
struct PcgAinvOp : OpBase {
    static constexpr bool STAGED = true, LOCAL = true;
    static constexpr int NRED = 2;
    const double *rOld, *w, *rD;
    double *rNew, *z;
    const SolverScalars *sc;
    Pre pre; // scalar step of the previous sweep, run in this kernel's prologue
    __device__ __forceinline__ bool prologue(const LayoutDev &) const { return pre.run(); }
    // the loads of stage() do not depend on one another: the engine issues a whole group of them before any use
    __device__ __forceinline__ double stage(int g) const
    {
        const double ro = rOld[g], ww = w[g], d = rD[g];
        const double r = sc->bodies > 0 ? fma(-sc->alpha, ww, ro) : ro;
        return __dmul_rn(d, r);
    }
    __device__ __forceinline__ double2 stage_own(int row) const
    {
        // rD is loaded before the store of rNew, which the compiler may not move a load past
        double2 r = *reinterpret_cast<const double2 *>(rOld + row);
        const double2 ww = *reinterpret_cast<const double2 *>(w + row);
        const double2 dd = *reinterpret_cast<const double2 *>(rD + row);
        if (sc->bodies > 0) {
            const double alpha = sc->alpha;
            r.x = fma(-alpha, ww.x, r.x);
            r.y = fma(-alpha, ww.y, r.y);
        }
        *reinterpret_cast<double2 *>(rNew + row) = r;
        return make_double2(__dmul_rn(dd.x, r.x), __dmul_rn(dd.y, r.y));
    }
    __device__ __forceinline__ double init(int, double) const { return 0.0; }
    __device__ __forceinline__ void finish(int row, double acc0, double acc1, double, double, double *red) const
    {
        // rNew[row] was written by this CTA in phase 1 (visible after the barrier)
        double2 d = *reinterpret_cast<const double2 *>(rD + row);
        double2 r = *reinterpret_cast<const double2 *>(rNew + row);
        double z0 = __dmul_rn(d.x, __dsub_rn(r.x, acc0));
        double z1 = __dmul_rn(d.y, __dsub_rn(r.y, acc1));
        *reinterpret_cast<double2 *>(z + row) = make_double2(z0, z1);
        red[0] += z0 * r.x + z1 * r.y;
        red[1] += fabs(r.x) + fabs(r.y);
    }
};

// K_B: applies the solution update of the PREVIOUS body (psi += alpha pOld, own rows, in
// place) and forms the new search direction while staging (p = z on the first body, else
// z + beta p; alpha, beta from the device scalars; p ping-ponged), then the row arithmetic
// of AmulOp<AMUL_OUT_X>: w = A p, fused <w,p>.  The halo send (fused pack CTAs) stages the same p at
// the patch face cells: stage() stays free of psi.
template <class Pre>
struct PcgAmulOp : AmulOp<AMUL_OUT_X> {
    const double *z, *pOld;
    double *pNew, *psi;
    const SolverScalars *sc;
    Pre pre; // scalar step of the previous sweep, run in this kernel's prologue
    __device__ __forceinline__ bool prologue(const LayoutDev &) const { return pre.run(); }
    // the loads of stage() do not depend on one another: the engine issues a whole group of them before any use
    __device__ __forceinline__ double stage(int g) const
    {
        const double zz = z[g], po = pOld[g];
        return sc->bodies == 0 ? zz : fma(sc->beta, po, zz);
    }
    __device__ __forceinline__ double2 stage_own(int row) const
    {
        // every load before the first store (the compiler may not move a load past a store to a vector that could
        // alias it): one memory round trip per row pair, not two (DESIGN §4)
        double2 zz = *reinterpret_cast<const double2 *>(z + row);
        const double2 po = *reinterpret_cast<const double2 *>(pOld + row);
        double2 x = *reinterpret_cast<const double2 *>(psi + row);
        if (sc->bodies > 0) {
            const double alpha = sc->alpha, beta = sc->beta;
            zz.x = fma(beta, po.x, zz.x);
            zz.y = fma(beta, po.y, zz.y);
            x.x = fma(alpha, po.x, x.x);
            x.y = fma(alpha, po.y, x.y);
            *reinterpret_cast<double2 *>(psi + row) = x;
        }
        *reinterpret_cast<double2 *>(pNew + row) = zz;
        return zz;
    }
};

// Close of the fused PCG: sweep A after the last body, without its preconditioner.  Runs the deferred step B of
// that body (its alpha) and sums |r| of r = rOld - alpha w into per-band partials grouped exactly as PcgAinvOp's sweep
// groups them (one CTA per band, lane k on rows 2k, 2k+1 of slices warp, warp + 8, ...), so the final residual keeps
// every bit; the <z,r> slot is 0.  r is not stored: nothing reads it after the solve.
template <class Pre>
__global__ void __launch_bounds__(ENGINE_THREADS) pcg_close_kernel(const LayoutDev L, const double *rOld,
                                                                    const double *w, const SolverScalars *sc,
                                                                    double *partials, Pre pre)
{
    if (!pre.run()) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double alpha = sc->alpha;
    double red[2] = {0, 0};
    for (int sl = warp; sl < L.slicesPerBand; sl += ENGINE_THREADS / 32) {
        const int row = blockIdx.x * L.bandRows + sl * SLICE_ROWS + 2 * lane;
        const double2 r = *reinterpret_cast<const double2 *>(rOld + row);
        const double2 ww = *reinterpret_cast<const double2 *>(w + row);
        red[1] += fabs(fma(-alpha, ww.x, r.x)) + fabs(fma(-alpha, ww.y, r.y));
    }
    block_reduce_store<2, ENGINE_THREADS>(red, partials, blockIdx.x);
}
