// solvers.cu -- lduMatrix::solver run-time selection and the Krylov / smooth solvers,
// running entirely on the device: alpha, beta and the convergence decision live in a
// device-resident SolverScalars block, every kernel of an iteration early-exits once
// the device has decided to stop, and the host only polls that flag every few
// iterations (pipelined, so polling never drains the GPU).  The iteration count and
// residual history are therefore exactly those of the reference's host-driven loop.
//
// Reference: LDU/lduMatrix/lduMatrixSolver.C:43-236 (selection, controls, normFactor),
// LDU/solvers/PCG/PCG.C:69-208, PBiCG/PBiCG.C:68-246, PBiCGStab/PBiCGStab.C:66-300,
// smoothSolver/smoothSolver.C:77-193, diagonalSolver/diagonalSolver.C:62-81,
// LduMatrix/LduMatrix/SolverPerformance.C:32-92.
#include "ldu.h"

#include <cstdlib>

#include "solver_steps.cuh"

// initial residual, normFactor and the first convergence test, common to all solvers
// (PCG.C:92-128; lduMatrixSolver.C:205-236).  wA must hold A.psi; tmp receives sumA.
int init_residual(Solve &S, const double *psi, const double *b, const double *wA, double *rA, double *tmp,
                  const double *wT, double *rT)
{
    SolverScalars *sc = S.sc;
    double *hist = S.hist;
    int np = 0;
    TRY(ew_launch<2>(S.ctx, S.n2, nullptr, S.partials, &np, [=] __device__(int i, double *red) {
        double2 bb = CV2(b)[i], ww = CV2(wA)[i], pp = CV2(psi)[i];
        double2 r = make_double2(__dsub_rn(bb.x, ww.x), __dsub_rn(bb.y, ww.y));
        V2(rA)[i] = r;
        if (rT) {
            double2 wt = CV2(wT)[i];
            V2(rT)[i] = make_double2(__dsub_rn(bb.x, wt.x), __dsub_rn(bb.y, wt.y));
        }
        red[0] += fabs(r.x) + fabs(r.y);
        red[1] += pp.x + pp.y;
    }));
    TRY(scalar_step<2>(S, np, [=] __device__(SolverScalars *s) {
        s->sumMag0 = s->sum[0];
        s->average = s->sum[1] / s->nCellsGlobal; // gAverage: gpuFieldCommonFunctions.C:611-635
    }));
    TRY(mat_sumA(S.m, tmp, nullptr));
    const int nCells = S.m->a->nCells;
    TRY(ew_launch<1>(S.ctx, S.n2, nullptr, S.partials, &np, [=] __device__(int i, double *red) {
        double avg = sc->average;
        double2 bb = CV2(b)[i], ww = CV2(wA)[i], tt = CV2(tmp)[i];
        double t0 = __dmul_rn(avg, tt.x), t1 = __dmul_rn(avg, tt.y);
        if (2 * i < nCells) red[0] += fabs(ww.x - t0) + fabs(bb.x - t0);
        if (2 * i + 1 < nCells) red[0] += fabs(ww.y - t1) + fabs(bb.y - t1);
    }));
    TRY(scalar_step<1>(S, np, [=] __device__(SolverScalars *s) {
        s->normFactor = s->sum[0] + SMALL_;
        s->initialResidual = s->sumMag0 / s->normFactor;
        s->finalResidual = s->initialResidual;
        hist_put(s, hist, 0, s->finalResidual);
        bool conv = check_convergence(s);
        if (!(s->minIter > 0 || !conv)) s->stop = 1;
    }));
    return B200LDU_OK;
}


// ---------------------------------------------------------------------------
// PCG (PCG.C:69-208)
// ---------------------------------------------------------------------------
int solve_pcg(Solve &S, int pk)
{
    b200ldu_matrix *m = S.m;
    SolverScalars *sc = S.sc;
    double *psi = S.psi, *b = S.src;
    double *pA = S.vec(0), *wA = S.vec(1), *rA = S.vec(2);
    if (!pA || !wA || !rA) return B200LDU_ECUDA;

    TRY(mat_amul(m, false, psi, wA, AMUL_ONLY, nullptr, nullptr, nullptr));
    TRY(init_residual(S, psi, b, wA, rA, pA));

    auto body = [&](long long) -> int {
        int np = 0;
        // wA = M^-1 rA ; wArA = <wA, rA>
        TRY(mat_precondition(m, pk, false, rA, wA, true, nullptr, S.partials, &np, S.stop));
        TRY(scalar_step<1>(S, np, BetaStep()));
        // pA = wA (first) | wA + beta*pA
        TRY(ew_launch<0>(S.ctx, S.n2, S.stop, nullptr, nullptr, [=] __device__(int i, double *) {
            double2 w = CV2(wA)[i];
            if (sc->nIterations == 0) {
                V2(pA)[i] = w;
            } else {
                double beta = sc->beta;
                double2 p = CV2(pA)[i];
                V2(pA)[i] = make_double2(fma(beta, p.x, w.x), fma(beta, p.y, w.y));
            }
        }));
        // wA = A pA ; wApA = <wA, pA>
        TRY(mat_amul(m, false, pA, wA, AMUL_OUT_X, nullptr, S.partials, S.stop));
        TRY(scalar_step<1>(S, S.nBands, AlphaStep()));
        // psi += alpha pA ; rA -= alpha wA ; sum|rA|
        TRY(ew_launch<1>(S.ctx, S.n2, S.stop, S.partials, &np, [=] __device__(int i, double *red) {
            double alpha = sc->alpha;
            double2 x = CV2(psi)[i], p = CV2(pA)[i], r = CV2(rA)[i], w = CV2(wA)[i];
            x.x = fma(alpha, p.x, x.x);
            x.y = fma(alpha, p.y, x.y);
            r.x = fma(-alpha, w.x, r.x);
            r.y = fma(-alpha, w.y, r.y);
            V2(psi)[i] = x;
            V2(rA)[i] = r;
            red[0] += fabs(r.x) + fabs(r.y);
        }));
        return scalar_step<1>(S, np, EndOfBody<0>{S.hist});
    };
    return run_iterations(S, max_bodies(S.c), body);
}

// ---------------------------------------------------------------------------
// PCG, fused form: TWO launches per iteration (the reference: 8 Thrust launches + 3 host synchronisations,
// PCG.C:131-205).  Sweep A (PcgAinvOp) applies the r update of the previous body while staging r,
// preconditions and reduces <z,r>, sum|r|; sweep B (PcgAmulOp) applies the psi update of the previous body and
// forms p = z + beta p while staging, multiplies and reduces <Ap,p>.  The scalar step that closes each sweep
// (sum of the per-band partials in fixed order, cross-rank all-reduce over the peer mailboxes, alpha / beta /
// convergence test) runs in the prologue of the NEXT sweep's kernel (ops.cuh DeferredStep) -- round 1 spent two
// one-CTA launches per iteration on it.  Same recurrences and per-row arithmetic as solve_pcg; the convergence
// decision of body k is taken at the start of sweep B of body k+1 (the preconditioner sweep that has then already
// run only overwrote scratch).  A solve that stops there leaves body k's psi update to the close.
// ---------------------------------------------------------------------------
// scalar step A of the fused PCG: closes body k-1 (residual, convergence: PCG.C:190-205), then beta of body k
struct PcgStepA {
    double *hist;
    __device__ void operator()(SolverScalars *s) const
    {
        if (s->bodies > 0) {
            EndOfBody<1>{hist}(s);
            if (s->stop) return;
        }
        s->psiBodies = s->bodies; // the sweep B this step opens adds the latest alpha p to psi
        BetaStep()(s);
    }
};
// scalar step B: alpha of body k
struct PcgStepB {
    __device__ void operator()(SolverScalars *s) const
    {
        if (AlphaStep()(s)) s->bodies++;
    }
};

int solve_pcg_fused(Solve &S, int pk)
{
    b200ldu_matrix *m = S.m;
    SolverScalars *sc = S.sc;
    const int *stop = S.stop;
    const int nBands = S.nBands;
    double *psi = S.psi, *b = S.src;
    double *pb[2] = {S.vec(0), S.vec(4)}, *w = S.vec(1), *rb[2] = {S.vec(2), S.vec(3)}, *z = S.vec(5);
    if (!pb[0] || !pb[1] || !w || !rb[0] || !rb[1] || !z) return B200LDU_ECUDA;
    const double *rD = m->d_rD;
    const P2PRed pr = (S.ctx->nRanks > 1 && S.ctx->p2p) ? comm_p2p_red(S.ctx) : P2PRed();
    // the two sweeps leave their partials in separate buffers: a deferred step reads one while the sweep that
    // runs it writes the other
    double *partA = S.partials, *partB = S.partials + 2 * (size_t)(nBands > S.ctx->smCount * 8 ? nBands : S.ctx->smCount * 8);

    TRY(mat_amul(m, false, psi, w, AMUL_ONLY, nullptr, nullptr, nullptr));
    TRY(init_residual(S, psi, b, w, rb[0], pb[0]));

    const PcgStepA gA{S.hist};
    const PcgStepB gB{};
    typedef DeferredStep<1, PcgStepB> PreA; // sweep A starts by closing sweep B of the previous body
    typedef DeferredStep<2, PcgStepA> PreB; // sweep B starts by closing sweep A of this body
    const int every = S.c.checkEvery > 0 ? S.c.checkEvery : 8;
    const unsigned mod = 2u * (unsigned)every;

    // diagonal / no preconditioner: sweep A is element-wise; its deferred step runs as CTA 0's prologue too
    auto sweepAew = [&](long long k, const PreA &preA, int *npA) -> int {
        const double *rOld = rb[k & 1];
        double *rNew = rb[(k + 1) & 1];
        return ew_launch<2>(S.ctx, S.n2, stop, partA, npA, [=] __device__(int i, double *red) {
            double2 r = CV2(rOld)[i];
            if (sc->bodies > 0) {
                const double alpha = sc->alpha;
                double2 ww = CV2(w)[i];
                r.x = fma(-alpha, ww.x, r.x);
                r.y = fma(-alpha, ww.y, r.y);
            }
            V2(rNew)[i] = r;
            double2 zz = r;
            if (pk == 1) {
                double2 d = CV2(rD)[i];
                zz = make_double2(__dmul_rn(d.x, r.x), __dmul_rn(d.y, r.y));
            }
            V2(z)[i] = zz;
            red[0] += zz.x * r.x + zz.y * r.y;
            red[1] += fabs(r.x) + fabs(r.y);
        }, preA);
    };
    auto preAFor = [&](long long k) {
        return PreA{partB, nBands, sc, gB, pr, (unsigned)(2 * (k % every)), mod, k > 0 ? 1 : 0};
    };

    auto body = [&](long long k) -> int {
        const double *rOld = rb[k & 1], *pPrev = pb[k & 1];
        double *rNew = rb[(k + 1) & 1], *pNew = pb[(k + 1) & 1];
        int npA = nBands;
        const PreA preA = preAFor(k);
        if (pk == 2) {
            PcgAinvOp<PreA> op;
            op.stop = stop;
            op.partials = partA;
            op.rOld = rOld, op.rNew = rNew, op.w = w, op.z = z, op.rD = m->d_rD;
            op.sc = sc;
            op.pre = preA;
            TRY(engine_launch_m(m, false, op));
        } else {
            TRY(sweepAew(k, preA, &npA));
        }
        int wait = 0;
        TRY(mat_halo(m, pNew, stop, &wait)); // peer-memory path: nothing is launched, the send is fused
        const PreB preB{partA, npA, sc, gA, pr, (unsigned)(2 * (k % every) + 1), mod, 1};
        PcgAmulOp<PreB> op{}; // zeroes the x and aux it inherits from AmulOp and does not read
        op.stop = stop;
        op.partials = partB;
        op.waitHalo = wait;
        op.z = z, op.pOld = pPrev, op.pNew = pNew, op.psi = psi, op.out = w, op.diag = m->d_diag;
        op.sc = sc;
        op.pre = preB;
        TRY(engine_launch_m(m, false, op));
        return B200LDU_OK;
    };
    const long long mb = max_bodies(S.c);
    TRY(run_iterations(S, mb, body));
    // Close, enqueued after the loop and never captured: the judgement of body mb-1 always stops the solve, so of the
    // sweep A that would follow only the deferred step B (alpha of body mb-1), r = rOld - alpha w and sum|r| are
    // needed; then the final EndOfBody.  All three are no-ops once the solve has stopped.  (mb is 0 only for a
    // negative maxIter: no body ran, nothing to close.)
    if (mb > 0) {
        int npA = nBands;
        if (pk == 2) {
            pcg_close_kernel<PreA><<<nBands, ENGINE_THREADS, 0, S.ctx->stream>>>(m->a->L, rb[mb & 1], w, sc, partA,
                                                                                 preAFor(mb));
            S.ctx->launches++;
            KERNEL_CHECK();
        } else {
            TRY(sweepAew(mb, preAFor(mb), &npA));
        }
        TRY(scalar_step_on<2>(S, partA, npA, EndOfBody<1>{S.hist}));
    }
    // The last alpha p that no sweep B added to psi (the solve stopped at a judgement, converged or not): exactly
    // one update, also after a stop, so the stop flag does not gate it.  p of body j lives in pb[(j + 1) & 1], and the
    // last alpha is body bodies-1's.
    const double *p0 = pb[0], *p1 = pb[1];
    return ew_launch<0>(S.ctx, S.n2, nullptr, nullptr, nullptr, [=] __device__(int i, double *) {
        const int j = sc->bodies;
        if (sc->psiBodies == j) return;
        const double alpha = sc->alpha;
        const double2 pp = CV2(j & 1 ? p1 : p0)[i], x = CV2(psi)[i];
        V2(psi)[i] = make_double2(fma(alpha, pp.x, x.x), fma(alpha, pp.y, x.y));
    });
}

// ---------------------------------------------------------------------------
// PBiCG (PBiCG.C:68-246)
// ---------------------------------------------------------------------------
int solve_pbicg(Solve &S, int pk)
{
    b200ldu_matrix *m = S.m;
    SolverScalars *sc = S.sc;
    double *psi = S.psi, *b = S.src;
    double *pA = S.vec(0), *wA = S.vec(1), *rA = S.vec(2), *pT = S.vec(3), *wT = S.vec(4), *rT = S.vec(5);
    if (!pA || !wA || !rA || !pT || !wT || !rT) return B200LDU_ECUDA;
    CUDA_TRY(cudaMemsetAsync(pT, 0, sizeof(double) * (size_t)m->a->vecLen, S.ctx->stream)); // pT = 0 :86

    TRY(mat_amul(m, false, psi, wA, AMUL_ONLY, nullptr, nullptr, nullptr));
    TRY(mat_amul(m, true, psi, wT, AMUL_ONLY, nullptr, nullptr, nullptr));
    TRY(init_residual(S, psi, b, wA, rA, pA, wT, rT));

    auto body = [&](long long) -> int {
        int np = 0;
        TRY(mat_precondition(m, pk, true, rT, wT, false, nullptr, nullptr, nullptr, S.stop));
        TRY(mat_precondition(m, pk, false, rA, wA, true, rT, S.partials, &np, S.stop)); // wArT = <wA, rT>
        TRY(scalar_step<1>(S, np, BetaStep()));
        TRY(ew_launch<0>(S.ctx, S.n2, S.stop, nullptr, nullptr, [=] __device__(int i, double *) {
            double2 w = CV2(wA)[i], wt = CV2(wT)[i];
            if (sc->nIterations == 0) {
                V2(pA)[i] = w;
                V2(pT)[i] = wt;
            } else {
                double beta = sc->beta;
                double2 p = CV2(pA)[i], pt = CV2(pT)[i];
                V2(pA)[i] = make_double2(fma(beta, p.x, w.x), fma(beta, p.y, w.y));
                V2(pT)[i] = make_double2(fma(beta, pt.x, wt.x), fma(beta, pt.y, wt.y));
            }
        }));
        TRY(mat_amul(m, true, pT, wT, AMUL_ONLY, nullptr, nullptr, S.stop));
        TRY(mat_amul(m, false, pA, wA, AMUL_OUT_AUX, pT, S.partials, S.stop)); // wApT = <wA, pT>
        TRY(scalar_step<1>(S, S.nBands, AlphaStep()));
        TRY(ew_launch<1>(S.ctx, S.n2, S.stop, S.partials, &np, [=] __device__(int i, double *red) {
            double alpha = sc->alpha;
            double2 x = CV2(psi)[i], p = CV2(pA)[i], r = CV2(rA)[i], w = CV2(wA)[i];
            double2 rt = CV2(rT)[i], wt = CV2(wT)[i];
            x.x = fma(alpha, p.x, x.x);
            x.y = fma(alpha, p.y, x.y);
            r.x = fma(-alpha, w.x, r.x);
            r.y = fma(-alpha, w.y, r.y);
            rt.x = fma(-alpha, wt.x, rt.x);
            rt.y = fma(-alpha, wt.y, rt.y);
            V2(psi)[i] = x;
            V2(rA)[i] = r;
            V2(rT)[i] = rt;
            red[0] += fabs(r.x) + fabs(r.y);
        }));
        return scalar_step<1>(S, np, EndOfBody<0>{S.hist});
    };
    return run_iterations(S, max_bodies(S.c), body);
}

// ---------------------------------------------------------------------------
// PBiCGStab (PBiCGStab.C:66-300)
// ---------------------------------------------------------------------------
int solve_pbicgstab(Solve &S, int pk)
{
    b200ldu_matrix *m = S.m;
    SolverScalars *sc = S.sc;
    double *hist = S.hist;
    const int quirk = S.c.bicgstabRefQuirk;
    double *psi = S.psi, *b = S.src;
    double *pA = S.vec(0), *yA = S.vec(1), *rA = S.vec(2), *AyA = S.vec(3), *sA = S.vec(4), *zA = S.vec(5),
           *tA = S.vec(6), *rA0 = S.vec(7);
    if (!pA || !yA || !rA || !AyA || !sA || !zA || !tA || !rA0) return B200LDU_ECUDA;

    TRY(mat_amul(m, false, psi, yA, AMUL_ONLY, nullptr, nullptr, nullptr));
    TRY(init_residual(S, psi, b, yA, rA, pA));
    CUDA_TRY(cudaMemcpyAsync(rA0, rA, sizeof(double) * (size_t)m->a->vecLen, cudaMemcpyDeviceToDevice,
                             S.ctx->stream)); // rA0 = rA :127

    auto body = [&](long long) -> int {
        int np = 0;
        // rA0rA = <rA0, rA>
        TRY(ew_launch<1>(S.ctx, S.n2, S.stop, S.partials, &np, [=] __device__(int i, double *red) {
            double2 x = CV2(rA0)[i], y = CV2(rA)[i];
            red[0] += x.x * y.x + x.y * y.y;
        }));
        TRY(scalar_step<1>(S, np, [=] __device__(SolverScalars *s) {
            s->rA0rAold = s->rA0rA;
            s->rA0rA = s->sum[0];
            if (!(fabs(s->rA0rA) > VSMALL_)) { // :141-144
                s->singular = 1;
                s->stop = 1;
                return;
            }
            if (s->nIterations > 0) {
                if (!(fabs(s->omega) > VSMALL_)) { // :153-156
                    s->singular = 1;
                    s->stop = 1;
                    return;
                }
                s->beta = (s->rA0rA / s->rA0rAold) * (s->alpha / s->omega);
            }
        }));
        // pA = rA (first) | rA + beta*(pA - omega*AyA)
        TRY(ew_launch<0>(S.ctx, S.n2, S.stop, nullptr, nullptr, [=] __device__(int i, double *) {
            double2 r = CV2(rA)[i];
            if (sc->nIterations == 0) {
                V2(pA)[i] = r;
            } else {
                double beta = sc->beta, omega = sc->omega;
                double2 p = CV2(pA)[i], ay = CV2(AyA)[i];
                double r1x = fma(-omega, ay.x, p.x), r1y = fma(-omega, ay.y, p.y);
                V2(pA)[i] = make_double2(fma(beta, r1x, r.x), fma(beta, r1y, r.y));
            }
        }));
        TRY(mat_precondition(m, pk, false, pA, yA, false, nullptr, nullptr, nullptr, S.stop));
        TRY(mat_amul(m, false, yA, AyA, AMUL_OUT_AUX, rA0, S.partials, S.stop)); // rA0AyA
        TRY(scalar_step<1>(S, S.nBands, [=] __device__(SolverScalars *s) { s->alpha = s->rA0rA / s->sum[0]; }));
        // sA = rA - alpha*AyA ; psi += alpha*yA (both exits of the body need it) ; sum|sA|
        TRY(ew_launch<1>(S.ctx, S.n2, S.stop, S.partials, &np, [=] __device__(int i, double *red) {
            double alpha = sc->alpha;
            double2 r = CV2(rA)[i], ay = CV2(AyA)[i], x = CV2(psi)[i], y = CV2(yA)[i];
            double2 s2 = make_double2(fma(-alpha, ay.x, r.x), fma(-alpha, ay.y, r.y));
            V2(sA)[i] = s2;
            V2(psi)[i] = make_double2(fma(alpha, y.x, x.x), fma(alpha, y.y, x.y));
            red[0] += fabs(s2.x) + fabs(s2.y);
        }));
        TRY(scalar_step<1>(S, np, [=] __device__(SolverScalars *s) {
            s->finalResidual = s->sum[0] / s->normFactor;
            if (check_convergence(s)) { // early return :198-213
                s->nIterations++;
                hist_put(s, hist, s->nIterations, s->finalResidual);
                s->stop = 1;
            }
        }));
        TRY(mat_precondition(m, pk, false, sA, zA, false, nullptr, nullptr, nullptr, S.stop));
        TRY(mat_amul(m, false, zA, tA, AMUL_OUT_OUT_OUT_AUX, sA, S.partials, S.stop)); // tAtA, tAsA
        TRY(scalar_step<2>(S, S.nBands, [=] __device__(SolverScalars *s) { s->omega = s->sum[1] / s->sum[0]; }));
        TRY(ew_launch<1>(S.ctx, S.n2, S.stop, S.partials, &np, [=] __device__(int i, double *red) {
            double omega = sc->omega;
            const double *second = quirk ? yA : zA; // PBiCGStab.C:263-270 passes yA
            double2 x = CV2(psi)[i], z = CV2(second)[i], s2 = CV2(sA)[i], t = CV2(tA)[i];
            V2(psi)[i] = make_double2(fma(omega, z.x, x.x), fma(omega, z.y, x.y));
            double2 r = make_double2(fma(-omega, t.x, s2.x), fma(-omega, t.y, s2.y));
            V2(rA)[i] = r;
            red[0] += fabs(r.x) + fabs(r.y);
        }));
        return scalar_step<1>(S, np, EndOfBody<0>{hist});
    };
    return run_iterations(S, max_bodies(S.c), body);
}

// ---------------------------------------------------------------------------
// smoothSolver (smoothSolver.C:77-193) with the Jacobi smoother
// ---------------------------------------------------------------------------
int solve_smooth(Solve &S)
{
    b200ldu_matrix *m = S.m;
    double *hist = S.hist;
    double *b = S.src;
    double *buf[2] = {S.psi, S.vec(0)};
    double *tmp = S.vec(1), *Apsi = S.vec(2);
    if (!buf[1] || !tmp || !Apsi) return B200LDU_ECUDA;
    const double omega = S.c.omega;
    const int nSweeps = S.c.nSweeps;
    // psi ping-pongs between buf[0] and buf[1], one sweep at a time; nIterations counts sweeps
    S.result = SolveResult{{buf[0], buf[1]}, 1, nSweeps > 0 ? nSweeps : 1};
    long long sweepsDone = 0;

    if (nSweeps < 0) { // fixed number of sweeps, no residual evaluation (:88-110); solve_banded seeded nIterations
        S.result.histEvery = 0;
        for (int s = 0; s < -nSweeps; s++, sweepsDone++)
            TRY(mat_jacobi(m, omega, buf[sweepsDone & 1], b, buf[(sweepsDone + 1) & 1], nullptr));
        return B200LDU_OK;
    }
    TRY(mat_amul(m, false, S.psi, Apsi, AMUL_ONLY, nullptr, nullptr, nullptr));
    TRY(init_residual(S, S.psi, b, Apsi, tmp, buf[1]));
    auto body = [&](long long) -> int {
        for (int s = 0; s < nSweeps; s++, sweepsDone++)
            TRY(mat_jacobi(m, omega, buf[sweepsDone & 1], b, buf[(sweepsDone + 1) & 1], S.stop));
        TRY(mat_residual(m, buf[sweepsDone & 1], b, tmp, true, S.partials, S.stop));
        return scalar_step<1>(S, S.nBands, [=] __device__(SolverScalars *s) {
            s->finalResidual = s->sum[0] / s->normFactor;
            int k = s->nIterations / (nSweeps > 0 ? nSweeps : 1) + 1;
            hist_put(s, hist, k, s->finalResidual);
            bool conv = check_convergence(s);
            s->nIterations += nSweeps; // ((nIterations += nSweeps) < maxIter && !conv) || nIterations < minIter
            bool cont = (s->nIterations < s->maxIter && !conv) || s->nIterations < s->minIter;
            if (!cont) s->stop = 1;
        });
    };
    int per = nSweeps > 0 ? nSweeps : 1;
    long long maxBodies = ((long long)(S.c.maxIter > S.c.minIter ? S.c.maxIter : S.c.minIter) + per - 1) / per + 1;
    return run_iterations(S, maxBodies, body);
}

// diagonalSolver.C:62-81; solve_banded seeded converged = 1
int solve_diagonal(Solve &S)
{
    const double *d = S.m->d_diag;
    double *psi = S.psi;
    const double *b = S.src;
    S.result.histEvery = 0;
    return ew_launch<0>(S.ctx, S.n2, nullptr, nullptr, nullptr, [=] __device__(int i, double *) {
        double2 bb = CV2(b)[i], dd = CV2(d)[i];
        V2(psi)[i] = make_double2(__ddiv_rn(bb.x, dd.x), __ddiv_rn(bb.y, dd.y));
    });
}

int gamg_solve(Solve &S, b200ldu_gamg *g); // gamg.cu

// ---------------------------------------------------------------------------
// the solve session
// ---------------------------------------------------------------------------
static thread_local int solveDepth = 0; // a solve nested in another one (GAMG coarsest level) polls its own flags

Solve::Solve(b200ldu_matrix *mat, const b200ldu_controls &controls, double *psi_b, double *src_b, int histCapacity,
             int nIterations0, int converged0)
    : m(mat), ctx(mat->a->ctx), sc((SolverScalars *)mat->d_scal), stop(&sc->stop), n2(mat->a->L.nPad / 2),
      nBands(mat->a->L.nBands), partials(mat->d_partials), psi(psi_b), src(src_b), c(controls), histCap(histCapacity)
{
    result.buf[0] = result.buf[1] = psi;
    rc = open(nIterations0, converged0);
}

int Solve::open(int nIterations0, int converged0)
{
    if (histCap > 0) TRY(m->mem.slot(MAT_HIST, hist, (size_t)histCap));
    entered_ = true;
    if (++solveDepth > SOLVE_MAX_DEPTH) {
        b200_set_error("solve: nesting too deep");
        return B200LDU_EINVAL;
    }
    pinnedFlags = ctx->pinned->flags[solveDepth - 1];
    pinnedFlags[0] = pinnedFlags[1] = 0;
    CUDA_TRY(cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&ev[1], cudaEventDisableTiming));

    // CUDA graphs need a capturable stream: if the context runs on the legacy default stream the
    // solve moves to the context's own stream, ordered against the caller's stream by events
    const char *env = getenv("B200LDU_GRAPH");
    useGraph = !(env && atoi(env) == 0) && (ctx->nRanks == 1 || ctx->p2p);
    if (useGraph && ctx->ownStream && ctx->stream != ctx->ownStream) {
        CUDA_TRY(cudaEventRecord(ev[0], ctx->stream));
        CUDA_TRY(cudaStreamWaitEvent(ctx->ownStream, ev[0], 0));
        userStream_ = ctx->stream;
        swapped_ = true;
        ctx->stream = ctx->ownStream;
    }

    const b200ldu_addr *a = m->a;
    SolverScalars h;
    memset(&h, 0, sizeof(h));
    h.wArA = GREAT_; // PCG.C:88
    h.wArAold = GREAT_;
    h.tolerance = c.tolerance;
    h.relTol = c.relTol;
    h.maxIter = c.maxIter;
    h.minIter = c.minIter;
    h.histCap = histCap;
    h.nSweeps = c.nSweeps;
    h.nCellsGlobal = a->nCellsGlobal > 0 ? a->nCellsGlobal : (double)a->nCells; // all-reduced at addr_create
    h.nIterations = nIterations0;
    h.converged = converged0;
    CUDA_TRY(cudaMemcpyAsync(sc, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
    return B200LDU_OK;
}

Solve::~Solve()
{
    if (swapped_) {
        if (cudaEventRecord(ev[0], ctx->ownStream) == cudaSuccess) cudaStreamWaitEvent(userStream_, ev[0], 0);
        ctx->stream = userStream_;
    }
    if (ev[0]) cudaEventDestroy(ev[0]);
    if (ev[1]) cudaEventDestroy(ev[1]);
    if (entered_) solveDepth--;
}

int Solve::finish(b200ldu_perf *perf, double *hist_h, double **psiOut)
{
    // read back the scalars (one synchronisation per solve)
    PinnedArea *pin = ctx->pinned;
    CUDA_TRY(cudaMemcpyAsync(&pin->scalars, sc, sizeof(SolverScalars), cudaMemcpyDeviceToHost, ctx->stream));
    pin->peerErr = 0;
    if (ctx->d_seq) // a bounded wait on a peer's flag gave up (engine.cuh spin_until)
        CUDA_TRY(cudaMemcpyAsync(&pin->peerErr, ctx->d_seq + 7, sizeof(pin->peerErr), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    int status = B200LDU_OK;
    if (pin->peerErr) {
        b200_set_error("solve: timed out waiting for a peer GPU's halo / all-reduce flag (a rank died or did not "
                       "enter the matching solve)");
        status = B200LDU_ENCCL;
    }
    const SolverScalars &h = pin->scalars;
    perf->initialResidual = h.initialResidual;
    perf->finalResidual = h.finalResidual;
    perf->normFactor = h.normFactor;
    perf->nIterations = h.nIterations;
    perf->converged = h.converged;
    perf->singular = h.singular;
    *psiOut = result.buf[((long long)h.nIterations * result.sweepsPerIteration) & 1];
    if (hist) {
        int k = result.histEvery > 0 ? h.nIterations / result.histEvery + 1 : 0;
        if (k > histCap) k = histCap;
        if (k > 0) CUDA_TRY(cudaMemcpy(hist_h, hist, sizeof(double) * (size_t)k, cudaMemcpyDeviceToHost));
        for (int i = k; i < histCap; i++) hist_h[i] = NAN;
    }
    return status;
}

// ---------------------------------------------------------------------------
// run-time selection: lduMatrixSolver.C:43-140
// ---------------------------------------------------------------------------
enum SolverBody { BODY_DIAGONAL, BODY_PCG, BODY_PCG_FUSED, BODY_PBICG, BODY_PBICGSTAB, BODY_SMOOTH, BODY_GAMG };

// The solver body to run, its preconditioner kind *pk and perf->solverName.  Allocates and enqueues nothing, so a
// refused selection leaves psi and the caller's history as they were.
static int select_solver(const b200ldu_matrix *m, const char *solver, const char *pre, const b200ldu_gamg *gamg,
                         b200ldu_perf *perf, SolverBody *body, int *pk)
{
    const b200ldu_addr *a = m->a;
    const char *sv = solver ? solver : "";
    if ((a->nFaces == 0 && a->L.nRecv == 0) || !strcmp(sv, "diagonal")) {
        strcpy(perf->solverName, "diagonal");
        *body = BODY_DIAGONAL;
        return B200LDU_OK;
    }
    // ICCG / BICCG wrappers (ICCG.C:40-51)
    if (!strcmp(sv, "ICCG")) {
        sv = "PCG";
        pre = "DIC";
    } else if (!strcmp(sv, "BICCG")) {
        sv = "PBiCG";
        pre = "DILU";
    }
    if (!strcmp(sv, "smoothSolver") || !strcmp(sv, "GAMG")) {
        if (!smoother_ok(pre)) return B200LDU_ENOPRECOND;
        *body = strcmp(sv, "GAMG") ? BODY_SMOOTH : BODY_GAMG;
        if (*body == BODY_GAMG && !gamg) {
            b200_set_error("GAMG needs an agglomeration handle (b200ldu_gamg_create)");
            return B200LDU_EINVAL;
        }
        strcpy(perf->solverName, sv);
        return B200LDU_OK;
    }
    if (strcmp(sv, "PCG") && strcmp(sv, "PBiCG") && strcmp(sv, "PBiCGStab")) {
        b200_set_error("Unknown %s solver %s; valid solvers: (BICCG GAMG ICCG PBiCG PBiCGStab PCG "
                       "diagonal smoothSolver)",
                       m->symmetric ? "symmetric" : "asymmetric", sv);
        return B200LDU_ENOSOLVER;
    }
    // solver::New looks the name up in the table of the matrix kind first (lduMatrixSolver.C:70-133); the
    // preconditioner is selected inside solve() from the tables of the same kind: DIC symmetric, DILU
    // asymmetric, AINV / diagonal / none both (DICPreconditioner.C:35, DILUPreconditioner.C:35, ...)
    const bool wantSym = !strcmp(sv, "PCG");
    char pname[32] = "";
    if (wantSym != (bool)m->symmetric) {
        b200_set_error("%s is registered for %s matrices only (PCG.C:36, PBiCG.C:36, PBiCGStab.C:36)", sv,
                       wantSym ? "symmetric" : "asymmetric");
        return B200LDU_EMATRIX;
    }
    if ((*pk = precond_kind(pre, pname)) < 0) return B200LDU_ENOPRECOND;
    if (pre && ((!strcmp(pre, "DILU") && m->symmetric) || (!strcmp(pre, "DIC") && !m->symmetric))) {
        b200_set_error("Unknown %s matrix preconditioner %s; valid %s matrix preconditioners: (AINV %s diagonal none)",
                       m->symmetric ? "symmetric" : "asymmetric", pre, m->symmetric ? "symmetric" : "asymmetric",
                       m->symmetric ? "DIC" : "DILU");
        return B200LDU_ENOPRECOND;
    }
    snprintf(perf->solverName, sizeof(perf->solverName), "%s%s", pname, sv);
    if (wantSym) {
        // the fused form needs every exchange inside the kernels: the peer-memory halo (or no halo)
        // and the peer-memory all-reduce (or one rank); otherwise -- cyclic patches, NCCL fall-back --
        // and with B200LDU_PCG_FUSED=0 the reference's op list runs kernel by kernel
        const char *ev = getenv("B200LDU_PCG_FUSED");
        const bool fused = !(ev && atoi(ev) == 0) && (a->L.nRecv == 0 || a->p2pHalo) &&
                           (a->ctx->nRanks == 1 || a->ctx->p2p);
        *body = fused ? BODY_PCG_FUSED : BODY_PCG;
    } else {
        *body = strcmp(sv, "PBiCG") ? BODY_PBICGSTAB : BODY_PBICG;
    }
    return B200LDU_OK;
}

// psi_b / src_b are banded vectors; *resultBuf receives the banded vector that holds the solution
int solve_banded(b200ldu_matrix *m, const char *solver, const char *pre, const b200ldu_controls *controls,
                 b200ldu_gamg *gamg, double *psi_b, double *src_b, b200ldu_perf *perf, double *hist_h,
                 int histCap, double **resultBuf)
{
    memset(perf, 0, sizeof(*perf));
    *resultBuf = psi_b;
    SolverBody body;
    int pk = 0;
    TRY(select_solver(m, solver, pre, gamg, perf, &body, &pk));
    b200ldu_controls c;
    if (controls)
        c = *controls;
    else
        b200ldu_controls_default(&c);
    // what the solvers that run no scalar step report: the diagonal solver converged, fixed sweeps count themselves
    const int nIterations0 = body == BODY_SMOOTH && c.nSweeps < 0 ? -c.nSweeps : 0;
    Solve S(m, c, psi_b, src_b, hist_h ? histCap : 0, nIterations0, body == BODY_DIAGONAL);
    TRY(S.rc);
    int rc = B200LDU_ECUDA;
    switch (body) {
    case BODY_DIAGONAL: rc = solve_diagonal(S); break;
    case BODY_PCG: rc = solve_pcg(S, pk); break;
    case BODY_PCG_FUSED: rc = solve_pcg_fused(S, pk); break;
    case BODY_PBICG: rc = solve_pbicg(S, pk); break;
    case BODY_PBICGSTAB: rc = solve_pbicgstab(S, pk); break;
    case BODY_SMOOTH: rc = solve_smooth(S); break;
    case BODY_GAMG: rc = gamg_solve(S, gamg); break;
    }
    if (rc != B200LDU_OK) {
        cudaStreamSynchronize(S.ctx->stream);
        return rc;
    }
    return S.finish(perf, hist_h, resultBuf);
}

extern "C" int b200ldu_solve(b200ldu_matrix *m, const char *solver, const char *pre,
                             const b200ldu_controls *controls, b200ldu_gamg *gamg, double *psi_d,
                             const double *source_d, b200ldu_perf *perf, double *hist_h, int histCap)
{
    if (!m || !psi_d || !source_d || !perf) {
        b200_set_error("solve: null argument");
        return B200LDU_EINVAL;
    }
    CUDA_TRY(cudaSetDevice(m->a->ctx->device));
    b200ldu_addr *a = m->a;
    // banded copies of psi and source live with the matrix workspace
    double *psi_b = banded_vec(a, m->mem, MAT_PSI), *src_b = banded_vec(a, m->mem, MAT_SRC);
    if (!psi_b || !src_b) return B200LDU_ECUDA;
    TRY(to_banded(a, psi_d, psi_b));
    TRY(to_banded(a, source_d, src_b));
    double *res = nullptr;
    TRY(solve_banded(m, solver, pre, controls, gamg, psi_b, src_b, perf, hist_h, histCap, &res));
    TRY(from_banded(a, res, psi_d));
    CUDA_TRY(cudaStreamSynchronize(a->ctx->stream));
    return B200LDU_OK;
}

extern "C" int b200ldu_solve_host(b200ldu_matrix *m, const char *solver, const char *pre,
                                  const b200ldu_controls *controls, b200ldu_gamg *gamg, double *psi_h,
                                  const double *source_h, b200ldu_perf *perf, double *hist_h, int histCap)
{
    if (!m || !psi_h || !source_h || !perf) {
        b200_set_error("solve_host: null argument");
        return B200LDU_EINVAL;
    }
    b200ldu_addr *a = m->a;
    b200ldu_ctx *ctx = a->ctx;
    CUDA_TRY(cudaSetDevice(ctx->device));
    size_t bytes = sizeof(double) * (size_t)a->nCells;
    double *psi_d = banded_vec(a, m->mem, MAT_HOST_PSI), *src_d = banded_vec(a, m->mem, MAT_HOST_SRC);
    if (!psi_d || !src_d) return B200LDU_ECUDA;
    // host buffers may be pageable: cudaMemcpyAsync then stages through the driver's pinned pool
    CUDA_TRY(cudaMemcpyAsync(psi_d, psi_h, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(src_d, source_h, bytes, cudaMemcpyHostToDevice, ctx->stream));
    TRY(b200ldu_solve(m, solver, pre, controls, gamg, psi_d, src_d, perf, hist_h, histCap));
    CUDA_TRY(cudaMemcpyAsync(psi_h, psi_d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return B200LDU_OK;
}
