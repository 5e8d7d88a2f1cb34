// mb200_kernels_std.cuh -- variable-state (STANDARD / morphological data) divisions: the reference's
// *_Std kernel family (CondLikeDown_Std src/likelihood.c:1920, CondLikeRoot_Std :4496,
// CondLikeScaler_Std :5547, Likelihood_Std :7359, TiProbs_Std :10066) as one fused pass.
//
// Every site pattern c has its own state count n_c = nStates[c] <= SMAX and its own run of K
// transition matrices inside a branch's block of matLen floats (tiIndex[c] + k * n_c^2).  In HBM the
// conditional likelihoods use the engine's padded layout [buf][k][c][Sp] (entries >= n_c are zero), so a
// (k, c) row is a few 16-byte loads; the host layout (mb200_get_partials) is the reference's ragged one.
//
// Thread mapping: one pattern = L = pow2ceil(K) adjacent lanes, one rate category each (the 4-state
// kernel's scheme): the rescaler's max over categories and the root's sum over categories are warp
// shuffles, nothing crosses a CTA.  A thread only ever re-reads rows it wrote itself, so a whole tree
// is walked in one launch without any barrier.  These divisions are small (hundreds of patterns): the
// pass is latency-bound, what matters is that it is ONE launch running beside the DNA partitions'.
//
// Arithmetic order is the reference's: like = sum_i P[a][i] * cl[i] from 0 upwards with separate
// multiply and add (the scalar C loops; the reference is built with -std=c99, i.e. no contraction),
// (likeL * likeR) * likeA, true divisions by the rescaler, (float) log (double) for the node scaler,
// double accumulation at the root.
#pragma once
#include "mb200_device.cuh"
#include <float.h>

#define MB200_BRLENS_MIN ((double)0.00000001f)   /* src/bayes.h:318 (float literal) */
#define MB200_BRLENS_MAX ((double)100.0f)        /* src/bayes.h:319                 */
#define MB200_STD_MAX_STATES 24                  /* MAX_STD_STATES, src/bayes.h:479 */

struct StdCtx                       // variable-state tables of an instance, passed by value
{
    const int  *nStates;            // [C]
    const int  *tiIndex;            // [C]
    const int  *bsIndex;            // [C]
    const int2 *classes;            // [nClasses] (state count, offset of its first matrix in a block)
    int         nClasses;
    int         matLen;             // floats per branch
    int         dummy;              // leading unobservable patterns
    int         uncompressed;       // sites the coding-bias correction applies to
    int         lanes;              // L: lanes per pattern
};

// ---------------------------------------------------------------------------------------
// K1 for the equal-frequency Mk model on unordered characters (TiProbs_Std, src/likelihood.c:10135-10173):
// pChange = 1/n - e/n, pNoChange = 1/n + (n-1)/n e, e = exp(-n/(n-1) v), v = length * rate_k with
// length clamped to [BRLENS_MIN, BRLENS_MAX] (:10125-10128).  grid = matrix updates, block = 64.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64)
tiprobs_std_kernel (DevCtx ctx, StdCtx sx, const DevEval *__restrict__ evals, int nEval, const double *__restrict__ dvals,
                    const DevMat *__restrict__ mats)
{
    __shared__ int sEvalIdx;
    const DevMat mu = mats[blockIdx.x];
    if (threadIdx.x == 0)
        sEvalIdx = owning_eval (evals, nEval, blockIdx.x);
    __syncthreads ();
    const double *rates = dvals + evals[sEvalIdx].dOff;
    double length = mu.length;
    if (length > MB200_BRLENS_MAX)      length = MB200_BRLENS_MAX;
    else if (length < MB200_BRLENS_MIN) length = MB200_BRLENS_MIN;
    float *block = ctx.matrices + (size_t)mu.matrix * sx.matLen;
    for (int q = threadIdx.x; q < sx.nClasses * ctx.K; q += blockDim.x)
        {
        const int2 cl = sx.classes[q / ctx.K];
        const int  k = q % ctx.K, n = cl.x;
        const double v = length * rates[k];
        const double eV1 = exp (-((double)n / ((double)n - 1.0)) * v);
        float pChange   = (float) ((1.0 / n) - ((1.0 / n) * eV1));
        const float pNoChange = (float) ((1.0 / n) + (((double)n - 1.0) / n) * eV1);
        if (pChange < 0.0f)
            pChange = 0.0f;
        float *P = block + cl.y + k * n * n;
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++)
                P[i*n + j] = (i == j) ? pNoChange : pChange;
        }
}

// ---------------------------------------------------------------------------------------
// fused pruning + rescaling + root integration.  grid = (pattern tiles, evaluations), block = NT.
// ---------------------------------------------------------------------------------------
template <int SMAX>
__device__ __forceinline__ void std_load_row (const DevCtx &ctx, int child, int c, int k, int n, float (&x)[SMAX])
{
    if (child < ctx.tipCount)
        {
        // tip conditional likelihoods: 1.0 for every state in the observed set (src/mcmc.c:6302-6330)
        const uint64_t m = ctx.tip64[(size_t)child * ctx.C + c];
        #pragma unroll
        for (int i = 0; i < SMAX; i++)
            x[i] = (i < n && ((m >> i) & 1)) ? 1.0f : 0.0f;
        }
    else
        {
        const float4 *src = reinterpret_cast<const float4 *>(ctx.partials + (size_t)(child - ctx.tipCount) * ((size_t)ctx.K * ctx.C * ctx.Sp)
                                                             + ((size_t)k * ctx.C + c) * ctx.Sp);
        #pragma unroll
        for (int q = 0; q < SMAX / 4; q++)
            {
            float4 t = make_float4 (0.0f, 0.0f, 0.0f, 0.0f);
            if (4*q < n)
                t = src[q];
            x[4*q] = t.x; x[4*q+1] = t.y; x[4*q+2] = t.z; x[4*q+3] = t.w;
            }
        }
}

template <int SMAX, int NT>
__global__ void __launch_bounds__(NT)
eval_std_kernel (DevCtx ctx, StdCtx sx, const DevEval *__restrict__ evals, const double *__restrict__ dvals,
                 const DevOp *__restrict__ ops, DevResult *out, int seq, int uniformMk)
{
    __shared__ double sSum[NT/32], sUn[NT/32];
    __shared__ int    sAb[NT/32];
    const int L = sx.lanes, TP = NT / L, K = ctx.K, C = ctx.C, Sp = ctx.Sp;
    const int p = threadIdx.x / L, k = threadIdx.x % L;
    const int c = blockIdx.x * TP + p;
    const bool act = (c < C) && (k < K);
    const bool lead = act && (k == 0);
    const DevEval *ev = evals + blockIdx.y;
    const int n = (c < C) ? sx.nStates[c] : 2;
    const int ti = (c < C) ? sx.tiIndex[c] : 0;
    const size_t bufStride = (size_t)K * C * Sp;
    const unsigned lane = threadIdx.x & 31u;
    const unsigned base = lane - (unsigned) k;                // first lane of this pattern's group

    float site = (act && ev->siteSrc >= 0) ? ctx.scalers[(size_t)ev->siteSrc * C + c] : 0.0f;
    float v[SMAX], x[SMAX];

    for (int o = 0; o < ev->nOp; o++)
        {
        const DevOp op = ops[ev->opOff + o];
        const int nChild = (op.c3 >= 0) ? 3 : 2;
        #pragma unroll 1
        for (int ch = 0; ch < nChild; ch++)
            {
            const int child = (ch == 0) ? op.c1 : (ch == 1) ? op.c2 : op.c3;
            const int mat   = (ch == 0) ? op.m1 : (ch == 1) ? op.m2 : op.m3;
            if (act)
                {
                std_load_row<SMAX> (ctx, child, c, k, n, x);
                const float *P = ctx.matrices + (size_t)mat * sx.matLen + ti + k * n * n;
                float pno = 0.0f, pch = 0.0f;
                if (uniformMk) { pno = P[0]; pch = P[1]; }        // Mk: two values per (state count, category)
                #pragma unroll
                for (int a = 0; a < SMAX; a++)
                    {
                    if (a < n)
                        {
                        float like = 0.0f;
                        #pragma unroll
                        for (int i = 0; i < SMAX; i++)
                            if (i < n)
                                {
                                const float pv = uniformMk ? ((i == a) ? pno : pch) : P[a*n + i];
                                like = __fadd_rn (like, __fmul_rn (pv, x[i]));
                                }
                        v[a] = (ch == 0) ? like : __fmul_rn (v[a], like);
                        }
                    else
                        v[a] = 0.0f;
                    }
                }
            }
        // RemoveNodeScalers (src/likelihood.c:7981-8002), CondLikeScaler_Std (:5547-5610)
        if (lead && op.sr >= 0)
            site -= ctx.scalers[(size_t)op.sr * C + c];
        if (op.sw >= 0)
            {
            float m = 0.0f;
            if (act)
                {
                #pragma unroll
                for (int a = 0; a < SMAX; a++)
                    if (a < n && v[a] > m)
                        m = v[a];
                }
            for (int off = 1; off < L; off <<= 1)
                m = fmaxf (m, __shfl_xor_sync (0xffffffffu, m, off));
            if (act)
                {
                #pragma unroll
                for (int a = 0; a < SMAX; a++)
                    if (a < n)
                        v[a] = __fdiv_rn (v[a], m);
                }
            if (lead)
                {
                const float sc = (float) log ((double) m);
                ctx.scalers[(size_t)op.sw * C + c] = sc;
                site += sc;
                }
            }
        if (act)
            {
            float4 *dst = reinterpret_cast<float4 *>(ctx.partials + (size_t)(op.dest - ctx.tipCount) * bufStride + ((size_t)k * C + c) * Sp);
            #pragma unroll
            for (int q = 0; q < SMAX / 4; q++)
                if (4*q < Sp)
                    dst[q] = make_float4 (v[4*q], v[4*q+1], v[4*q+2], v[4*q+3]);
            }
        }

    if (lead && ev->siteDst >= 0)
        ctx.scalers[(size_t)ev->siteDst * C + c] = site;
    if (ev->root < 0)
        return;

    // ---- Likelihood_Std, numBetaCats == 1 (src/likelihood.c:7401-7455): like = sum_k (sum_j cl * bs) / K ----
    double catTerm = 0.0;
    if (act)
        {
        std_load_row<SMAX> (ctx, ev->root, c, k, n, x);
        const double *bs = dvals + ev->dOff + 2*K + sx.bsIndex[c];
        double catLike = 0.0;
        #pragma unroll
        for (int j = 0; j < SMAX; j++)
            if (j < n)
                catLike += (double) x[j] * bs[j];
        catTerm = catLike * (1.0 / (double) K);
        }
    double like = 0.0;
    for (int kk = 0; kk < K; kk++)                              // the reference's order over categories
        like += __shfl_sync (0xffffffffu, catTerm, base + kk);
    double term = 0.0, pUn = 0.0; int abortFlag = 0;
    if (lead)
        {
        if (c < sx.dummy)
            pUn = like * exp ((double) site);                   // unobservable pattern: feeds the coding-bias correction
        else if (like < MB200_LIKE_EPSILON)
            abortFlag = 1;
        else
            term = ((double) site + log (like)) * (double) ctx.weights[(size_t)ev->weightsRow * C + c];
        }

    // ---- deterministic reduction: lanes, warps, then the tiles in order by the last CTA to arrive ----
    #pragma unroll
    for (int off = 16; off > 0; off >>= 1)
        {
        term      += __shfl_xor_sync (0xffffffffu, term, off);
        pUn       += __shfl_xor_sync (0xffffffffu, pUn, off);
        abortFlag |= __shfl_xor_sync (0xffffffffu, abortFlag, off);
        }
    if (lane == 0) { sSum[threadIdx.x >> 5] = term; sUn[threadIdx.x >> 5] = pUn; sAb[threadIdx.x >> 5] = abortFlag; }
    __syncthreads ();
    if (threadIdx.x == 0)
        {
        double s = 0.0, u = 0.0; int a = 0;
        #pragma unroll
        for (int w = 0; w < NT/32; w++) { s += sSum[w]; u += sUn[w]; a |= sAb[w]; }
        if (tile_arrive (ctx, blockIdx.y, ctx.numTiles, blockIdx.x, make_double2 (s, u), a))
            {
            const TileSum ts = tile_sum_ltr (ctx, blockIdx.y, ctx.numTiles);
            // correct for absent characters (src/likelihood.c:7417-7423, 7537)
            double pObserved = 1.0 - ts.unobserved;
            if (pObserved < MB200_LIKE_EPSILON)
                pObserved = MB200_LIKE_EPSILON;
            const double tot = ts.lnL - log (pObserved) * (double) sx.uncompressed;
            dev_result_write (&out[blockIdx.y], ts.abort ? -DBL_MAX : tot, ts.abort ? 1 : 0, seq);
            }
        }
}
