// mb200_kernels_tcp.cuh -- warp-specialised, pipelined wgmma pruning kernel (eval_tcp_kernel) for the 20-state
// amino-acid and 61-state codon paths (CondLikeDown/Root_Gen*, _NY98*, CondLikeScaler_Gen*, Likelihood_Gen*/_NY98*;
// reference src/likelihood.c:204, 1575, 2152, 4010, 4939, 5413, 5764, 6975).
//
// Work = (node, 128-pattern tile) items of the device-side queue of mb200_kernels_tc.cuh (level order, acquire /
// release flags between the CTAs of a persistent grid).  Inside the CTA the phases of an item do not run back to
// back: one CTA per SM, 18 warps with fixed roles, mbarrier rings between them.
//
//   scheduler (1 warp)    draws tickets, decodes (slot, evaluation, tile), waits for the item's producers (flag
//                         acquire), publishes the item in a 4-deep shared-memory ring
//   loaders   (8 warps)   one *unit* = one (rate category, child) operand of an item.  Groups of warps take the units
//                         round-robin, so several units' loads are in flight per SM: child rows HBM/L2 -> registers
//                         (512-byte coalesced LDG.128) -> hi/lo TF32 split -> canonical K-major core-matrix images in
//                         an operand-ring stage; the branch's pre-split P(t) image [hi | lo] arrives in the same stage by
//                         one bulk async copy (TMA engine, complete_tx on the stage's full barrier)
//   consumers (2 x 4)     two warpgroups, one per 64-row half of the tile.  Per unit: [main | corr] = A_hi x [B_hi | B_lo]^T
//                         (ONE wgmma chain, N = 2 NP) and corr += A_lo x B_hi^T (N = NP), accumulators in registers; once
//                         the MMAs have completed the operand stage goes back to the loaders.  Then main + corr, product
//                         over the children (kept in the shared-memory staging area), row maximum; after the last child
//                         coalesced 16-byte stores of row * (1 / max) -- the two roundings of the reference's rescaler;
//                         node scaler; the evaluation's closing item (site scalers, root integration, lnL tile sums)
//                         runs here too
//   publisher (1 warp)    release-stores the node-done flags (the memory barrier of a release does not stall a warp that
//                         has the next item's operands waiting)
//
// 3xTF32 as before (x = hi + lo, lo x lo dropped); the large term and the two correction terms land in separate
// accumulators and are added in FP32 in the epilogue.
#pragma once
#include "mb200_kernels_tc.cuh"

template <int S> struct TcpGeom;
// LG: loader groups (8 / LG warps each) -- units go round-robin to the groups, so LG units' loads are in flight per SM;
// a 20-state unit is small (30 KB), hence more, smaller groups
template <> struct TcpGeom<61> { static constexpr int LG = 2; };
template <> struct TcpGeom<20> { static constexpr int LG = 4; };

constexpr int TCP_THREADS   = 576;     // 2 x 4 consumer warps, 8 loader warps, scheduler, publisher
constexpr int TCP_NPUB      = 4;       // flag-publication ring (epilogue -> publisher warp)
constexpr int TCP_NS_MAX    = 8;       // operand-ring stages (as many as fit beside the staging area)
constexpr int TCP_NI        = 4;       // item ring
constexpr int TCP_ITEM_NODE = 0, TCP_ITEM_CLOSE = 1, TCP_ITEM_STOP = 2;

struct TcpItem                          // 64 bytes
{
    int kind, e, t, oi;
    int nChild, dest, sw, shortcut;
    int child[3], mat[3];
    int pad[2];
};

template <int S> __host__ __device__ constexpr size_t tcp_stage_bytes ()
{
    return (size_t)(2 * 128 * TcGeom<S>::KP + 2 * TcGeom<S>::NP * TcGeom<S>::KP) * sizeof(float);
}
template <int S> __host__ __device__ constexpr size_t tcp_staging_bytes (int K)
{
    return (size_t) K * ((S + 3) / 4) * 129 * sizeof(float4);   // one item's result rows, [k][16-byte chunk][row + pad]
}
// "this row's tip is fully ambiguous" bytes, one 128-byte record per operand-ring stage (loader -> consumers; read
// before the stage is handed back)
template <int S> __host__ __device__ constexpr size_t tcp_tipring_bytes (int NS) { return (size_t) NS * 128; }
// stages that fit in `limit` bytes of dynamic shared memory: a multiple of the loader groups (every stage is then
// always filled by the same group, which sees each of its phases -- the parity wait cannot alias), or 1: one group
// loads everything
template <int S> inline int tcp_stages (int K, size_t limit)
{
    const size_t st = tcp_staging_bytes<S> (K) + tcp_tipring_bytes<S> (0);
    if (st + tcp_stage_bytes<S> () + 128 > limit) return 0;
    size_t n = (limit - st) / (tcp_stage_bytes<S> () + 128);
    if (n > (size_t) TCP_NS_MAX) n = TCP_NS_MAX;
    if (n >= (size_t) TcpGeom<S>::LG) n -= n % TcpGeom<S>::LG;
    else if (n >= 2) n = 2;
    return (int) n;
}

// mbarrier wait that cannot hang the device: a CTA whose pipeline stalls for two seconds traps (the launch fails
// with an error instead of sitting on the GPU until somebody's watchdog fires)
__device__ __forceinline__ void tcp_wait (uint64_t *bar, uint32_t parity)
{
    const uint32_t a = gmma::smem_u32 (bar);
    uint32_t done = 0;
    unsigned long long t0 = 0;
    for (unsigned it = 0; ; it++)
        {
        asm volatile ("{\n\t.reg .pred p;\n\t"
                      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                      "selp.u32 %0, 1, 0, p;\n\t}\n" : "=r"(done) : "r"(a), "r"(parity) : "memory");
        if (done) return;
        __nanosleep (32);                      // a waiting warp must not compete for issue slots with the working ones
        if ((it & 0xfffu) == 0xfffu)
            {
            unsigned long long now;
            asm volatile ("mov.u64 %0, %%globaltimer;\n" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 2000000000ull) __trap ();
            }
        }
}
__device__ __forceinline__ void tcp_bar_epilogue () { asm volatile ("bar.sync 3, 256;\n" ::: "memory"); }      // both epilogue halves
// barrier of one epilogue half (warps 0-3: id 1, warps 4-7: id 2)
__device__ __forceinline__ void tcp_bar_group (int grp)
{
    if (grp == 0) asm volatile ("bar.sync 1, 128;\n" ::: "memory");
    else          asm volatile ("bar.sync 2, 128;\n" ::: "memory");
}

template <int S>
__global__ void __launch_bounds__(TCP_THREADS, 1)
eval_tcp_kernel (DevCtx ctx, TcQueue Q, int NS, const DevEval *__restrict__ evals, const double *__restrict__ dvals,
                 const DevOp *__restrict__ ops, const float *__restrict__ split, DevResult *out, int seq)
{
    using namespace gmma;
    constexpr int NP = TcGeom<S>::NP, KP = TcGeom<S>::KP;
    constexpr int TM = 128;
    constexpr uint32_t LBO_A = (TM / 8) * 128, LBO_B = (2 * NP / 8) * 128, SBO = 128;
    constexpr int A_FLOATS = TM * KP;
    constexpr int B_FLOATS = 2 * NP * KP;
    constexpr int NQ = (S + 3) / 4;
    constexpr int SPC = TcGeom<S>::SP;
    constexpr size_t STAGE = tcp_stage_bytes<S> ();

    extern __shared__ __align__(128) unsigned char tcp_smem[];
    __shared__ uint64_t barFull[TCP_NS_MAX], barEmpty[TCP_NS_MAX], barInfoFull[TCP_NI], barInfoEmpty[TCP_NI];
    __shared__ TcpItem sInfo[TCP_NI];
    __shared__ uint64_t barPubFull[TCP_NPUB], barPubEmpty[TCP_NPUB];
    __shared__ int   *sPub[TCP_NPUB];  // flags to release, in order (nullptr: stop)
    __shared__ float  sMax[TM];        // row maxima (each row belongs to one consumer warpgroup)
    __shared__ double qSum[2][4];
    __shared__ int    qAb[2][4];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int Sp = ctx.Sp, K = ctx.K, C = ctx.C;
    float4 *sStage = reinterpret_cast<float4 *>(tcp_smem + (size_t) NS * STAGE);     // [k][chunk][TM+1]
    const int TIPRING = NS;
    unsigned char *sTipFull = tcp_smem + (size_t) NS * STAGE + tcp_staging_bytes<S> (K);   // [unit % TIPRING][row]

    if (tid == 32)
        {
        for (int s = 0; s < NS; s++) { mbar_init (&barFull[s], 8 / TcpGeom<S>::LG + 1); mbar_init (&barEmpty[s], 8); }
        for (int i = 0; i < TCP_NI; i++) { mbar_init (&barInfoFull[i], 1); mbar_init (&barInfoEmpty[i], 16); }
        for (int i = 0; i < TCP_NPUB; i++) { mbar_init (&barPubFull[i], 1); mbar_init (&barPubEmpty[i], 1); }
        mbar_fence_init ();
        }
    __syncthreads ();
    const size_t bufStride = (size_t)K * C * Sp;
    const int rows = TM, numTiles = ctx.numTiles;
    const int perSlot = Q.nEval * numTiles;
    const int total = (Q.maxOps + 1) * perSlot;

    if (warp == 16)
        {
        // =================================================================== scheduler
        int slot = 0; uint32_t ph = 0;
        for (;;)
            {
            tcp_wait (&barInfoEmpty[slot], ph ^ 1);
            int item = 0;
            if (lane == 0) item = (int)(atomicAdd (Q.counter, 1u) - Q.base);
            item = __shfl_sync (0xffffffffu, item, 0);
            TcpItem it;
            it.kind = TCP_ITEM_STOP; it.e = it.t = it.oi = 0; it.nChild = 0; it.dest = it.sw = -1; it.shortcut = 0;
            it.child[0] = it.child[1] = it.child[2] = -1; it.mat[0] = it.mat[1] = it.mat[2] = -1; it.pad[0] = it.pad[1] = 0;
            if (item >= 0 && item < total)
                {
                const int sl = item / perSlot, e = (item % perSlot) / numTiles, t = item % numTiles;
                const DevEval *ev = evals + e;
                const int nOp = ev->nOp;
                if (sl > nOp)
                    continue;                                   // shorter evaluation: nothing in this slot
                const int *flagRow = Q.flags + ((size_t)e * numTiles + t) * Q.flagStride;
                it.e = e; it.t = t;
                if (sl < nOp)
                    {
                    const int   oi = Q.order[ev->opOff + sl];
                    const DevOp op = ops[ev->opOff + oi];
                    it.kind = TCP_ITEM_NODE; it.oi = oi;
                    it.nChild = (op.c3 >= 0) ? 3 : 2; it.dest = op.dest; it.sw = op.sw;
                    it.shortcut = (ev->flags & MB200_SHORTCUT_FLAG) ? 1 : 0;
                    it.child[0] = op.c1; it.child[1] = op.c2; it.child[2] = op.c3;
                    it.mat[0] = op.m1; it.mat[1] = op.m2; it.mat[2] = op.m3;
                    if (lane < 3)
                        {
                        const int pr = (lane == 0) ? op.s1 : (lane == 1) ? op.s2 : op.s3;
                        if (pr >= 0)
                            {
                            unsigned spins = 0;
                            while (tcq_ld_acquire (flagRow + pr) != seq)
                                {
                                __nanosleep (64);
                                if ((++spins & 1023u) == 0 && (spins > (1u << 22) || *((volatile int *) Q.error)))
                                    { *Q.error = 1; break; }                    // bounded: never hang the device
                                }
                            }
                        }
                    }
                else
                    {
                    it.kind = TCP_ITEM_CLOSE;
                    for (int o = lane; o < nOp; o += 32)
                        {
                        unsigned spins = 0;
                        while (tcq_ld_acquire (flagRow + o) != seq)
                            {
                            __nanosleep (128);
                            if ((++spins & 1023u) == 0 && (spins > (1u << 22) || *((volatile int *) Q.error)))
                                { *Q.error = 1; break; }
                            }
                        }
                    }
                __syncwarp ();
                }
            if (lane == 0)
                {
                sInfo[slot] = it;
                mbar_arrive (&barInfoFull[slot]);              // release: the record is visible to whoever acquires the phase
                }
            if (it.kind == TCP_ITEM_STOP)
                break;
            if (++slot == TCP_NI) { slot = 0; ph ^= 1; }
            }
        }
    else if (warp >= 8 && warp < 16)
        {
        // =================================================================== loaders: groups of warps, units round-robin
        constexpr int LGMAX = TcpGeom<S>::LG, WPG = 8 / LGMAX;     // warps per group
        const int nGroups = (NS >= LGMAX) ? LGMAX : (NS >= 2) ? 2 : 1;          // NS is a multiple of nGroups
        const int grp = (warp - 8) / WPG, lw = (warp - 8) % WPG, ltid = lw * 32 + lane;
        constexpr int QB = (KP / 4 + 3) / 4;                    // chunk blocks of 4 per row
        constexpr int NIT = (TM / 8) * QB / WPG;                // items per thread and unit
        constexpr int TPR = TM / (WPG * 32);                    // tip rows per thread
        const uint64_t fullMaskL = (S == 64) ? ~(uint64_t)0 : ((((uint64_t)1) << S) - 1);
        int islot = 0; uint32_t iph = 0;
        unsigned u = 0;                                         // units since the kernel started (all roles count alike)
        for (;;)
            {
            tcp_wait (&barInfoFull[islot], iph);
            const int kind = sInfo[islot].kind, tileIdx = sInfo[islot].t, nChild = sInfo[islot].nChild;
            const int ch0 = sInfo[islot].child[0], ch1 = sInfo[islot].child[1], ch2 = sInfo[islot].child[2];
            const int mt0 = sInfo[islot].mat[0], mt1 = sInfo[islot].mat[1], mt2 = sInfo[islot].mat[2];
            __syncwarp ();
            if (lane == 0) mbar_arrive (&barInfoEmpty[islot]);
            if (++islot == TCP_NI) { islot = 0; iph ^= 1; }
            if (kind == TCP_ITEM_STOP) break;
            if (kind == TCP_ITEM_CLOSE) continue;
            const int c0 = tileIdx * rows, np = min (rows, C - c0);
            for (int k = 0; k < K; k++)
                for (int ch = 0; ch < nChild; ch++, u++)
                    {
                    if ((int)(u % (unsigned) nGroups) != grp)
                        continue;
                    const int s = (int)(u % (unsigned) NS);
                    const uint32_t ph = (u / (unsigned) NS) & 1u;
                    const int child = (ch == 0) ? ch0 : (ch == 1) ? ch1 : ch2, mat = (ch == 0) ? mt0 : (ch == 1) ? mt1 : mt2;
                    const bool isTip = child < ctx.tipCount;
                    unsigned char *stg = tcp_smem + (size_t) s * STAGE;
                    float4 x[NIT];
                    uint64_t m[TPR];
                    int partAmbig = 0;
                    // loads first, then the wait for the stage: the round trip overlaps the MMAs still reading it
                    if (isTip)
                        {
                        partAmbig = ctx.tipPartAmbig[child];
                        #pragma unroll
                        for (int j = 0; j < TPR; j++)
                            {
                            const int r = ltid + j * (WPG * 32);
                            m[j] = (r < np) ? ctx.tip64[(size_t)child * C + c0 + r] : 0;
                            }
                        }
                    else
                        {
                        const float *src = ctx.partials + (size_t)(child - ctx.tipCount) * bufStride + ((size_t)k * C + c0) * Sp;
                        #pragma unroll
                        for (int n = 0; n < NIT; n++)
                            {
                            const int i2 = lw + WPG * n;
                            const int rb = i2 / QB, qb = i2 % QB;
                            const int r = rb * 8 + (lane & 7), q = qb * 4 + (lane >> 3);
                            x[n] = make_float4 (0.f, 0.f, 0.f, 0.f);
                            if (q < KP / 4 && r < np && q * 4 < SPC)
                                x[n] = __ldcg (reinterpret_cast<const float4 *>(src + (size_t)r * SPC + q * 4));
                            }
                        }
                    tcp_wait (&barEmpty[s], ph ^ 1);
                    if (ltid == 0)
                        {
                        mbar_expect_tx (&barFull[s], (uint32_t)(B_FLOATS * 4));
                        bulk_g2s (stg + 2 * A_FLOATS * 4, split + ((size_t)mat * K + k) * B_FLOATS, (uint32_t)(B_FLOATS * 4), &barFull[s]);
                        }
                    if (isTip)
                        {
                        // thread = row(s): the state mask expands to 0/1 (exact in TF32; no lo image); the epilogue
                        // learns through the tip ring which rows see a fully ambiguous tip (preLike shortcut)
                        #pragma unroll
                        for (int j = 0; j < TPR; j++)
                            {
                            const int r = ltid + j * (WPG * 32);
                            sTipFull[(u % (unsigned) TIPRING) * 128 + r] = (m[j] == fullMaskL && !partAmbig) ? 1 : 0;
                            #pragma unroll
                            for (int q = 0; q < KP / 4; q++)
                                {
                                float4 h;
                                h.x = ((m[j] >> (q*4 + 0)) & 1) ? 1.f : 0.f; h.y = ((m[j] >> (q*4 + 1)) & 1) ? 1.f : 0.f;
                                h.z = ((m[j] >> (q*4 + 2)) & 1) ? 1.f : 0.f; h.w = ((m[j] >> (q*4 + 3)) & 1) ? 1.f : 0.f;
                                *reinterpret_cast<float4 *>(stg + canon_off (r, q*4, TM)) = h;
                                }
                            }
                        }
                    else
                        {
                        #pragma unroll
                        for (int n = 0; n < NIT; n++)
                            {
                            const int i2 = lw + WPG * n;
                            const int rb = i2 / QB, qb = i2 % QB;
                            const int r = rb * 8 + (lane & 7), q = qb * 4 + (lane >> 3);
                            if (q < KP / 4)
                                {
                                const float4 h = make_float4 (to_tf32 (x[n].x), to_tf32 (x[n].y), to_tf32 (x[n].z), to_tf32 (x[n].w));
                                const float4 l = make_float4 (to_tf32 (x[n].x - h.x), to_tf32 (x[n].y - h.y), to_tf32 (x[n].z - h.z), to_tf32 (x[n].w - h.w));
                                *reinterpret_cast<float4 *>(stg + canon_off (r, q*4, TM)) = h;
                                *reinterpret_cast<float4 *>(stg + A_FLOATS * 4 + canon_off (r, q*4, TM)) = l;
                                }
                            }
                        }
                    fence_async_smem ();                        // generic-proxy stores -> async proxy (wgmma)
                    __syncwarp ();
                    if (lane == 0) mbar_arrive (&barFull[s]);
                    }
            }
        }
    else if (warp == 17)
        {
        // =================================================================== publisher: release-stores the node-done flags,
        // so that no epilogue warp sits in a memory barrier
        int slot = 0; uint32_t ph = 0;
        for (;;)
            {
            tcp_wait (&barPubFull[slot], ph);
            int *flag = sPub[slot];
            __syncwarp ();
            if (lane == 0)
                {
                mbar_arrive (&barPubEmpty[slot]);
                if (flag != nullptr)
                    tcq_st_release (flag, seq);                // fence + store: everything the epilogue wrote is visible first
                }
            if (flag == nullptr)
                break;
            if (++slot == TCP_NPUB) { slot = 0; ph ^= 1; }
            }
        }
    else
        {
        // =================================================================== consumers: warpgroup g = rows [64 g, 64 g + 64)
        // of every item.  The products are staged UNSCALED in shared memory ([k][chunk][row]), the row maxima meet in
        // sMax, and all 256 threads copy the rows out with coalesced 16-byte stores of row * (1 / max) -- the two
        // roundings of CondLikeScaler_Gen (src/likelihood.c:4939-4990).
        constexpr uint64_t A_LO = (A_FLOATS * 4) >> 4, A_KS = (2 * LBO_A) >> 4, B_KS = (2 * LBO_B) >> 4;
        const int grp = warp >> 2, gtid = tid & (TM - 1), row = gtid;
        const int fRow = grp * 64 + (warp & 3) * 16 + (lane >> 2), fCol = 2 * (lane & 3);   // accumulator fragment
        int islot = 0; uint32_t iph = 0;
        int pslot = 0; uint32_t pph = 0;
        unsigned u = 0;
        for (;;)
            {
            tcp_wait (&barInfoFull[islot], iph);
            struct { int kind, e, t, oi, nChild, dest, sw, shortcut; } it;
            it.kind = sInfo[islot].kind; it.e = sInfo[islot].e; it.t = sInfo[islot].t; it.oi = sInfo[islot].oi;
            it.nChild = sInfo[islot].nChild; it.dest = sInfo[islot].dest; it.sw = sInfo[islot].sw; it.shortcut = sInfo[islot].shortcut;
            const int ch0 = sInfo[islot].child[0], ch1 = sInfo[islot].child[1], ch2 = sInfo[islot].child[2];
            __syncwarp ();
            if (lane == 0) mbar_arrive (&barInfoEmpty[islot]);
            if (++islot == TCP_NI) { islot = 0; iph ^= 1; }
            if (it.kind == TCP_ITEM_STOP)
                {
                if (tid == 0)
                    {
                    tcp_wait (&barPubEmpty[pslot], pph ^ 1);
                    sPub[pslot] = nullptr;
                    mbar_arrive (&barPubFull[pslot]);
                    }
                break;
                }
            const int   c0 = it.t * rows, np = min (rows, C - c0);
            const int   c  = c0 + row;
            const bool  active = row < np;
            const DevEval *ev = evals + it.e;
            int *flagRow = Q.flags + ((size_t)it.e * numTiles + it.t) * Q.flagStride;

            if (it.kind == TCP_ITEM_NODE)
                {
                float mx[2] = { 0.0f, 0.0f };                   // fragment rows fRow, fRow + 8
                for (int k = 0; k < K; k++)
                    for (int ch = 0; ch < it.nChild; ch++, u++)
                        {
                        const int s = (int)(u % (unsigned) NS);
                        const int child = (ch == 0) ? ch0 : (ch == 1) ? ch1 : ch2;
                        const bool isTip = child < ctx.tipCount;
                        tcp_wait (&barFull[s], (u / (unsigned) NS) & 1u);   // operand images (generic stores + bulk copy) have landed
                        const uint32_t st = smem_u32 (tcp_smem + (size_t) s * STAGE);
                        const uint64_t aHi = make_desc (st + grp * (64 / 8) * 128, LBO_A, SBO), aLo = aHi + A_LO;
                        const uint64_t bb  = make_desc (st + 2 * A_FLOATS * 4, LBO_B, SBO);
                        float acc[NP];                          // [main | corr] columns of this thread's fragment
                        #pragma unroll
                        for (int i = 0; i < NP; i++) { acc[i] = 0.0f; fence_regs (acc[i]); }
                        mma_fence ();
                        #pragma unroll
                        for (int ks = 0; ks < KP / 8; ks++)
                            mma_tf32<2 * NP> (acc, aHi + ks * A_KS, bb + ks * B_KS, ks > 0);
                        if (!isTip)
                            {
                            #pragma unroll
                            for (int ks = 0; ks < KP / 8; ks++)
                                mma_tf32<NP> (acc + NP / 2, aLo + ks * A_KS, bb + ks * B_KS, true);
                            }
                        mma_commit ();
                        mma_wait_all ();
                        #pragma unroll
                        for (int i = 0; i < NP; i++) fence_regs (acc[i]);
                        // preLike shortcut of the scalar kernels (src/likelihood.c:257-258): a fully ambiguous tip contributes exactly 1
                        bool tipFull[2] = { false, false };
                        if (it.shortcut && isTip)
                            {
                            tipFull[0] = sTipFull[(u % (unsigned) TIPRING) * 128 + fRow] != 0;
                            tipFull[1] = sTipFull[(u % (unsigned) TIPRING) * 128 + fRow + 8] != 0;
                            }
                        __syncwarp ();
                        if (lane == 0) mbar_arrive (&barEmpty[s]);     // operands read: the stage goes back to the loaders
                        const bool last = ch == it.nChild - 1;
                        #pragma unroll
                        for (int j = 0; j < NP / 8; j++)
                            {
                            const int col = 8 * j + fCol;
                            if (col >= 4 * NQ) continue;        // padding columns beyond the staged chunks
                            #pragma unroll
                            for (int h = 0; h < 2; h++)
                                {
                                float v0 = acc[4 * j + 2 * h] + acc[NP / 2 + 4 * j + 2 * h];
                                float v1 = acc[4 * j + 2 * h + 1] + acc[NP / 2 + 4 * j + 2 * h + 1];
                                if (tipFull[h]) { v0 = 1.0f; v1 = 1.0f; }
                                float2 *p = reinterpret_cast<float2 *>(reinterpret_cast<float *>(sStage) +
                                                                       (((size_t)k * NQ + col / 4) * (TM + 1) + fRow + 8 * h) * 4 + (col & 3));
                                if (ch > 0)
                                    {
                                    const float2 o = *p;        // product of the earlier children (this thread wrote it)
                                    v0 = o.x * v0; v1 = o.y * v1;
                                    }
                                if (last)
                                    {
                                    if (col >= S) v0 = 0.0f;
                                    if (col + 1 >= S) v1 = 0.0f;
                                    mx[h] = fmaxf (mx[h], fmaxf (v0, v1));
                                    }
                                *p = make_float2 (v0, v1);
                                }
                            }
                        }
                #pragma unroll
                for (int h = 0; h < 2; h++)
                    {
                    mx[h] = fmaxf (mx[h], __shfl_xor_sync (0xffffffffu, mx[h], 1));
                    mx[h] = fmaxf (mx[h], __shfl_xor_sync (0xffffffffu, mx[h], 2));
                    }
                if ((lane & 3) == 0) { sMax[fRow] = mx[0]; sMax[fRow + 8] = mx[1]; }
                // the warpgroups meet: row maxima, then the copy-out
                tcp_bar_epilogue ();
                const bool doScale = it.sw >= 0;
                {
                float *dstBase = ctx.partials + (size_t)(it.dest - ctx.tipCount) * bufStride;
                constexpr int nq = SPC / 4, NCP = (nq + 1) / 2;
                // the reciprocals of the rows this thread copies, all of them first (straight-line code below: the
                // shared-memory loads of the copy are then in flight together)
                float fr[NCP];
                #pragma unroll
                for (int n = 0; n < NCP; n++)
                    {
                    const int idx = n * 256 + tid;
                    const int r = (idx < nq * TM) ? idx / nq : 0;
                    fr[n] = doScale ? __frcp_rn (sMax[r]) : 1.0f;      // = 1.0f / max, IEEE
                    }
                for (int k = 0; k < K; k++)
                    {
                    float4 *dst = reinterpret_cast<float4 *>(dstBase + ((size_t)k * C + c0) * SPC);
                    float4 v[NCP];
                    #pragma unroll
                    for (int n = 0; n < NCP; n++)
                        {
                        const int idx = n * 256 + tid;
                        const int r = (idx < nq * TM) ? idx / nq : 0, q = idx % nq;
                        v[n] = sStage[((size_t)k * NQ + ((q < NQ) ? q : 0)) * (TM + 1) + r];
                        if (q >= NQ) v[n] = make_float4 (0.f, 0.f, 0.f, 0.f);
                        }
                    #pragma unroll
                    for (int n = 0; n < NCP; n++)
                        {
                        const int idx = n * 256 + tid;
                        const int r = idx / nq;
                        v[n].x *= fr[n]; v[n].y *= fr[n]; v[n].z *= fr[n]; v[n].w *= fr[n];
                        if (r < np && idx < nq * TM)
                            dst[idx] = v[n];
                        }
                    }
                }
                if (doScale && grp == 0 && active)              // node scaler (CondLikeScaler_Gen_SSE: log in double, cast to float, src/likelihood.c:5055)
                    ctx.scalers[(size_t)it.sw * C + c] = log_of_max (sMax[row]);
                // publish: the barrier orders every epilogue thread's stores before thread 0's hand-over; the publisher warp
                // acquires it and release-stores the flag (cumulative at GPU scope), so no epilogue warp sits in a memory
                // barrier while the next item's accumulators are waiting
                tcp_bar_epilogue ();
                if (tid == 0)
                    {
                    tcp_wait (&barPubEmpty[pslot], pph ^ 1);
                    sPub[pslot] = flagRow + it.oi;
                    mbar_arrive (&barPubFull[pslot]);
                    if (++pslot == TCP_NPUB) { pslot = 0; pph ^= 1; }
                    }
                continue;
                }

            // ---------------------------------------------------------------- closing item of (e, t): warps 0-3
            if (grp != 0)
                continue;
            const int nOp = ev->nOp;
            float site = 0.0f;
            if (active)
                {
                site = (ev->siteSrc >= 0) ? ctx.scalers[(size_t)ev->siteSrc * C + c] : 0.0f;
                for (int o = 0; o < nOp; o++)                  // the caller's operation order (src/likelihood.c:7938-7965)
                    {
                    const DevOp op = ops[ev->opOff + o];
                    if (op.sr >= 0) site -= __ldcg (ctx.scalers + (size_t)op.sr * C + c);
                    if (op.sw >= 0) site += __ldcg (ctx.scalers + (size_t)op.sw * C + c);
                    }
                if (ev->siteDst >= 0)
                    ctx.scalers[(size_t)ev->siteDst * C + c] = site;
                }
            if (ev->root < 0)
                continue;
            double term = 0.0; int abortFlag = 0;
            if (active)
                {
                const double *rates = dvals + ev->dOff;
                const double *catW = rates + K, *freqs = rates + 2*K;
                const float *rootBase = ctx.partials + (size_t)(ev->root - ctx.tipCount) * bufStride;
                double like = 0.0;
                for (int k = 0; k < K; k++)
                    {
                    const float4 *rp = reinterpret_cast<const float4 *>(rootBase + ((size_t)k * C + c) * Sp);
                    double s = 0.0;
                    #pragma unroll 4
                    for (int q = 0; q < NQ; q++)
                        {
                        const float4 v = __ldcg (rp + q);
                        s += (double) v.x * freqs[q*4];
                        if (q*4 + 1 < S) s += (double) v.y * freqs[q*4 + 1];
                        if (q*4 + 2 < S) s += (double) v.z * freqs[q*4 + 2];
                        if (q*4 + 3 < S) s += (double) v.w * freqs[q*4 + 3];
                        }
                    like += s * catW[k];
                    }
                double likeI = 0.0;
                if (ev->hasPInvar)
                    {
                    const uint64_t im = ctx.invMask[c];
                    for (int i = 0; i < S; i++)
                        if ((im >> i) & 1) likeI += freqs[i];
                    likeI *= ev->pInvar;
                    }
                term = site_term (like, likeI, ev->hasPInvar, ev->flags & MB200_QUIRK_FLAG, site,
                                  ctx.weights[(size_t)ev->weightsRow * C + c], abortFlag);
                }
            // tile partial -> ticket -> the last tile of the evaluation adds the partials in tile order
            #pragma unroll
            for (int off = 16; off > 0; off >>= 1)
                {
                term      += __shfl_xor_sync (0xffffffffu, term, off);
                abortFlag |= __shfl_xor_sync (0xffffffffu, abortFlag, off);
                }
            if (lane == 0) { qSum[grp][warp & 3] = term; qAb[grp][warp & 3] = abortFlag; }
            tcp_bar_group (grp);
            if (gtid == 0)
                {
                const double s = qSum[grp][0] + qSum[grp][1] + qSum[grp][2] + qSum[grp][3];
                const int    a = qAb[grp][0] | qAb[grp][1] | qAb[grp][2] | qAb[grp][3];
                if (tile_arrive (ctx, it.e, numTiles, it.t, make_double2 (s, 0.0), a))
                    {
                    const TileSum ts = tile_sum_ltr (ctx, it.e, numTiles);
                    const int ab = ts.abort | *((volatile int *) Q.error);
                    dev_result_write (&out[it.e], ab ? -DBL_MAX : ts.lnL, ab ? 1 : 0, seq);
                    }
                }
            tcp_bar_group (grp);                               // qSum / qAb free for the group's next closing item
            }
        }

}
