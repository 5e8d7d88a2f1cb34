/*
 * pruning_oracle.c -- TEST INFRASTRUCTURE (see pruning_oracle.h): plain-C restatement of the
 * reference's tree-likelihood path.  Each function cites the reference code it follows.
 * Compiled with -ffp-contract=off so that every float multiply/add rounds exactly where the
 * reference's intrinsics round; fused operations are written explicitly with fmaf().
 *
 * Layouts are the reference's scalar ones: CL [k][c][s] (src/mcmc.c:5756, 6397-6413),
 * P [k][i][j] (src/likelihood.c:300-309), scalers [c], cijk block [lambda_re, lambda_im, c_ijk]
 * (src/likelihood.c:9467-9468).  Tips are kept as state-set masks and expanded to the 0/1
 * vectors the reference stores (src/mcmc.c:6350-6413).
 */
#include "pruning_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define ORC_MAX_INST 256
#define ORC_TIME_MIN ((double)1.0E-11f)   /* src/bayes.h:321 (float literal) */
#define ORC_TIME_MAX ((double)100.0f)     /* src/bayes.h:322                 */
#define ORC_LIKE_EPSILON 1.0e-300         /* src/likelihood.c:44             */

typedef struct
    {
    mb200_instance_config cfg;
    int         arith;
    uint64_t   *tips;        /* [tip][C]                                             */
    int        *tipPartAmbig;/* [tip]: some pattern neither single state nor missing  */
    float      *partials;    /* [interior buffer][K][C][S]                           */
    float      *matrices;    /* [matrix][K][S][S]                                    */
    float      *scalers;     /* [scaler][C]                                          */
    double     *eigen;       /* [slot][parts][2S+S^3]                                */
    int         parts;       /* eigensystems per slot (1, or K for NY98-type models)  */
    float      *weights;     /* [row][C]                                             */
    float      *tmp[3];      /* per-child matvec results [K][C][S]                   */
    long long   updates;
    int         guardHit;       /* MB200_FLAG_RANGE_GUARD tripped during the evaluation in progress */
    /* variable-state (STANDARD data) divisions: the *_Std family */
    int         std;         /* MB200_CONFIG_VARIABLE_STATES                          */
    int        *nStates, *tiIndex, *bsIndex;    /* [C] m->nStates, m->tiIndex, m->bsIndex */
    size_t     *clOff;       /* [C+1] offset of pattern c inside one category's block  */
    int         matLen, dummy, uncompressed;
    } OrcInst;

static OrcInst *orcTab[ORC_MAX_INST];

static OrcInst *Get (int id)
{
    if (id < 0 || id >= ORC_MAX_INST)
        return NULL;
    return orcTab[id];
}

int orc_create_instance (const mb200_instance_config *c, int *instance)
{
    int     id, i;
    size_t  S, K, C, nInt;
    OrcInst *o;

    if (!c || !instance)
        return MB200_ERROR_GENERAL;
    if (c->state_count < 2 || c->state_count > MB200_MAX_STATES || c->category_count < 1 ||
        c->category_count > MB200_MAX_CATEGORIES || c->pattern_count < 1 || c->tip_count < 2 ||
        c->partials_count <= c->tip_count)
        return MB200_ERROR_OUT_OF_RANGE;
    for (id=0; id<ORC_MAX_INST; id++)
        if (orcTab[id] == NULL)
            break;
    if (id == ORC_MAX_INST)
        return MB200_ERROR_OUT_OF_MEMORY;
    o = (OrcInst *) calloc (1, sizeof(OrcInst));
    o->cfg = *c;
    o->arith = ORC_ARITH_FMA;
    S = (size_t)c->state_count; K = (size_t)c->category_count; C = (size_t)c->pattern_count;
    nInt = (size_t)(c->partials_count - c->tip_count);
    o->tips         = (uint64_t *) calloc ((size_t)c->tip_count * C, sizeof(uint64_t));
    o->tipPartAmbig = (int *)      calloc ((size_t)c->tip_count, sizeof(int));
    o->partials     = (float *)    calloc (nInt * K * C * S, sizeof(float));
    o->matrices     = (float *)    calloc ((size_t)c->matrix_count * K * S * S, sizeof(float));
    o->scalers      = (float *)    calloc ((size_t)c->scaler_count * C, sizeof(float));
    o->parts        = (((c->flags >> 8) & 0xff) > 1) ? ((c->flags >> 8) & 0xff) : 1;
    o->eigen        = (double *)   calloc ((size_t)c->eigen_count * o->parts * (2*S + S*S*S), sizeof(double));
    o->weights      = (float *)    calloc ((size_t)c->weight_rows * C, sizeof(float));
    for (i=0; i<3; i++)
        o->tmp[i]   = (float *)    calloc (K * C * S, sizeof(float));
    o->std = (c->flags & MB200_CONFIG_VARIABLE_STATES) ? 1 : 0;
    orcTab[id] = o;
    *instance = id;
    return MB200_SUCCESS;
}

int orc_finalize_instance (int instance)
{
    int i;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    free (o->tips); free (o->tipPartAmbig); free (o->partials); free (o->matrices);
    free (o->scalers); free (o->eigen); free (o->weights);
    free (o->nStates); free (o->tiIndex); free (o->bsIndex); free (o->clOff);
    for (i=0; i<3; i++) free (o->tmp[i]);
    free (o);
    orcTab[instance] = NULL;
    return MB200_SUCCESS;
}

int orc_set_arith (int instance, int arith)
{
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    o->arith = arith;
    return MB200_SUCCESS;
}

long long orc_cl_updates (int instance)
{
    OrcInst *o = Get (instance);
    return o ? o->updates : 0;
}

/* tip codes; isPartAmbig as SetUpTermState decides it (src/mcmc.c:18631-18651) */
int orc_set_tip_states (int instance, int tip, const uint64_t *masks)
{
    int c, C, S;
    uint64_t full, m;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (tip < 0 || tip >= o->cfg.tip_count || !masks) return MB200_ERROR_OUT_OF_RANGE;
    C = o->cfg.pattern_count; S = o->cfg.state_count;
    full = (S == 64) ? ~(uint64_t)0 : (((uint64_t)1 << S) - 1);
    o->tipPartAmbig[tip] = 0;
    for (c=0; c<C; c++)
        {
        m = masks[c] & full;
        o->tips[(size_t)tip*C + c] = m;
        if (m != full && (m == 0 || (m & (m - 1)) != 0))
            o->tipPartAmbig[tip] = 1;
        }
    return MB200_SUCCESS;
}

int orc_set_pattern_weights (int instance, int row, const float *w)
{
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (row < 0 || row >= o->cfg.weight_rows || !w) return MB200_ERROR_OUT_OF_RANGE;
    memcpy (o->weights + (size_t)row * o->cfg.pattern_count, w, (size_t)o->cfg.pattern_count * sizeof(float));
    return MB200_SUCCESS;
}

int orc_set_cijk (int instance, int eigen, const double *block)
{
    size_t S, n;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (eigen < 0 || eigen >= o->cfg.eigen_count || !block) return MB200_ERROR_OUT_OF_RANGE;
    S = (size_t)o->cfg.state_count; n = (size_t)o->parts * (2*S + S*S*S);
    memcpy (o->eigen + (size_t)eigen * n, block, n * sizeof(double));
    return MB200_SUCCESS;
}

/* CalcCijk (src/utils.c:9734-9746): c[i][j][k] = u[i][k] * v[k][j] */
int orc_set_eigen_decomposition (int instance, int eigen, const double *u, const double *v, const double *lam)
{
    size_t S, n, i, j, k;
    double *b, *pc;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (eigen < 0 || eigen >= o->cfg.eigen_count || !u || !v || !lam) return MB200_ERROR_OUT_OF_RANGE;
    if (o->parts != 1) return MB200_ERROR_UNSUPPORTED;
    S = (size_t)o->cfg.state_count; n = 2*S + S*S*S;
    b = o->eigen + (size_t)eigen * n;
    for (i=0; i<S; i++) { b[i] = lam[i]; b[S+i] = 0.0; }
    pc = b + 2*S;
    for (i=0; i<S; i++)
        for (j=0; j<S; j++)
            for (k=0; k<S; k++)
                *pc++ = u[i*S+k] * v[k*S+j];
    return MB200_SUCCESS;
}

/* TiProbs_Gen (src/likelihood.c:9499-9542) for one branch */
static void TiProbs (OrcInst *o, const mb200_matrix_update *mu, const mb200_evaluation *ev)
{
    int     S = o->cfg.state_count, K = o->cfg.category_count, i, j, k, s, index;
    double  t, sum, e[MB200_MAX_STATES];
    const size_t partLen = 2*(size_t)S + (size_t)S*S*S;
    const double *lam0 = (mu->eigen == MB200_EIGEN_INLINE) ? ev->inline_eigen
                                                           : o->eigen + (size_t)mu->eigen * o->parts * partLen;
    const double *lam = lam0;
    const double *ptr;
    float  *tiP = o->matrices + (size_t)mu->matrix * K * S * S;

    for (k=index=0; k<K; k++)
        {
        /* TiProbs_GenCov (src/likelihood.c:9568-9690): one eigensystem per category */
        lam = lam0 + ((o->parts > 1) ? (size_t)k * partLen : 0);
        t = mu->length * ev->category_rates[k];
        if (t < ORC_TIME_MIN)
            {
            for (i=0; i<S; i++)
                for (j=0; j<S; j++)
                    tiP[index++] = (i == j) ? 1.0f : 0.0f;
            }
        else if (t > ORC_TIME_MAX)
            {
            for (i=0; i<S; i++)
                for (j=0; j<S; j++)
                    tiP[index++] = (float) ev->state_freqs[j];
            }
        else
            {
            for (s=0; s<S; s++)
                e[s] = exp (lam[s] * t);
            ptr = lam + 2*S;
            for (i=0; i<S; i++)
                for (j=0; j<S; j++)
                    {
                    sum = 0.0;
                    for (s=0; s<S; s++)
                        sum += (*ptr++) * e[s];
                    tiP[index++] = (float) ((sum < 0.0) ? 0.0 : sum);
                    }
            }
        }
}

/* one child's contribution q[k][c][i] = sum_j P_k[i][j] * cl[k][c][j]
 * interior / dense tips: CondLikeDown_Gen case 0 (src/likelihood.c:298-318) and
 *   CondLikeDown_NUC4_FMA (src/likelihood.c:1147-1169) for the fused variant;
 * tips without partial ambiguity when shortcuts apply: the preLike tables
 *   (src/likelihood.c:236-260): a single observed state copies the P column, a missing
 *   observation contributes exactly 1.0 */
static void ChildTerm (OrcInst *o, int child, int matrix, int shortcuts, float *out)
{
    int     S = o->cfg.state_count, K = o->cfg.category_count, C = o->cfg.pattern_count, c, i, j, k;
    const float *P, *cl;
    float   x[MB200_MAX_STATES], acc;
    uint64_t full = (S == 64) ? ~(uint64_t)0 : (((uint64_t)1 << S) - 1), m;
    int     isTip = child < o->cfg.tip_count;
    int     useShort = isTip && shortcuts && !o->tipPartAmbig[child];

    for (k=0; k<K; k++)
        {
        P = o->matrices + ((size_t)matrix * K + k) * S * S;
        for (c=0; c<C; c++)
            {
            float *dst = out + ((size_t)k*C + c)*S;
            if (isTip)
                {
                m = o->tips[(size_t)child*C + c];
                if (useShort && m == full)
                    {
                    for (i=0; i<S; i++) dst[i] = 1.0f;
                    continue;
                    }
                for (j=0; j<S; j++) x[j] = ((m >> j) & 1) ? 1.0f : 0.0f;
                cl = x;
                }
            else
                cl = o->partials + ((size_t)(child - o->cfg.tip_count)*K + k)*C*S + (size_t)c*S;
            for (i=0; i<S; i++)
                {
                const float *row = P + (size_t)i*S;
                if (o->arith == ORC_ARITH_FMA && S == 4)
                    {
                    acc = row[0] * cl[0];
                    acc = fmaf (row[1], cl[1], acc);
                    acc = fmaf (row[2], cl[2], acc);
                    acc = fmaf (row[3], cl[3], acc);
                    }
                else if (S == 4)
                    {
                    /* CondLikeDown_NUC4_SSE / _AVX: first product, then mul + add */
                    acc = row[0] * cl[0];
                    acc = row[1] * cl[1] + acc;
                    acc = row[2] * cl[2] + acc;
                    acc = row[3] * cl[3] + acc;
                    }
                else
                    {
                    acc = 0.0f;
                    for (j=0; j<S; j++)
                        acc = row[j] * cl[j] + acc;
                    }
                dst[i] = acc;
                }
            }
        }
}

/* one interior node: CondLikeDown / CondLikeRoot, RemoveNodeScalers, CondLikeScaler
 * (src/likelihood.c:7920-7965) */
static void Operation (OrcInst *o, const mb200_operation *op, const mb200_evaluation *ev, float *lnScaler)
{
    int     S = o->cfg.state_count, K = o->cfg.category_count, C = o->cfg.pattern_count, c, k, s;
    size_t  n = (size_t)K * C * S, idx;
    int     shortcuts = (ev->flags & MB200_FLAG_TIP_SHORTCUTS) != 0;
    float  *dst = o->partials + (size_t)(op->dest - o->cfg.tip_count) * n;
    float   scaler, *scP;

    ChildTerm (o, op->child1, op->matrix1, shortcuts, o->tmp[0]);
    ChildTerm (o, op->child2, op->matrix2, shortcuts, o->tmp[1]);
    if (op->child3 != MB200_NONE)
        {
        ChildTerm (o, op->child3, op->matrix3, shortcuts, o->tmp[2]);
        for (idx=0; idx<n; idx++)
            dst[idx] = o->tmp[0][idx] * o->tmp[1][idx] * o->tmp[2][idx];
        }
    else
        {
        for (idx=0; idx<n; idx++)
            dst[idx] = o->tmp[0][idx] * o->tmp[1][idx];
        }
    o->updates += (long long) K * C;

    /* RemoveNodeScalers (src/likelihood.c:7981-8002) */
    if (op->scale_remove != MB200_NONE && lnScaler)
        {
        scP = o->scalers + (size_t)op->scale_remove * C;
        for (c=0; c<C; c++)
            lnScaler[c] -= scP[c];
        }
    /* CondLikeScaler_* (src/likelihood.c:4939-4990, 5202-5262) */
    if (op->scale_write != MB200_NONE)
        {
        scP = o->scalers + (size_t)op->scale_write * C;
        for (c=0; c<C; c++)
            {
            scaler = 0.0f;
            for (k=0; k<K; k++)
                for (s=0; s<S; s++)
                    if (dst[((size_t)k*C + c)*S + s] > scaler)
                        scaler = dst[((size_t)k*C + c)*S + s];
            for (k=0; k<K; k++)
                for (s=0; s<S; s++)
                    dst[((size_t)k*C + c)*S + s] /= scaler;
            if (o->arith == ORC_ARITH_FMA && S == 4)
                scP[c] = logf (scaler);              /* CondLikeScaler_NUC4_AVX :5257 */
            else
                scP[c] = (float) log (scaler);       /* _Gen_SSE :5055, _NUC4_SSE :5328 */
            if (lnScaler)
                lnScaler[c] += scP[c];
            if ((ev->flags & MB200_FLAG_RANGE_GUARD) && S == 4 && scaler < 1.0e-24f)
                o->guardHit = 1;                     /* MB200_FLAG_RANGE_GUARD (include/mb200.h): 4-state only */
            }
        }
}

/* Likelihood_NUC4_{FMA,SSE} (src/likelihood.c:6468-6625, 6804-6960) and
 * Likelihood_Gen_SSE / Likelihood_Gen (src/likelihood.c:5926-6090, 5764-5916) */
static int RootLikelihood (OrcInst *o, const mb200_evaluation *ev, const float *lnScaler, double *lnL)
{
    int     S = o->cfg.state_count, K = o->cfg.category_count, C = o->cfg.pattern_count, c, k, s, t, equal = 1;
    size_t  n = (size_t)K * C * S;
    const float *cl = o->partials + (size_t)(ev->root_buffer - o->cfg.tip_count) * n;
    const float *w = o->weights + (size_t)ev->weights_row * C;
    float   bs[MB200_MAX_STATES], likeF, catLike, likeIF;
    double  like, likeI, lnLike, sum = 0.0;
    uint64_t inv;
    int     quirk = (ev->flags & MB200_FLAG_NUC4_PINVAR_QUIRK) != 0;

    for (s=0; s<S; s++) bs[s] = (float) ev->state_freqs[s];
    for (k=1; k<K; k++) if (ev->category_weights[k] != ev->category_weights[0]) equal = 0;

    for (c=0; c<C; c++)
        {
        if (S == 4 && equal)
            {
            likeF = 0.0f;
            for (k=0; k<K; k++)
                for (s=0; s<4; s++)
                    {
                    if (o->arith == ORC_ARITH_FMA)
                        likeF = fmaf (cl[((size_t)k*C + c)*4 + s], bs[s], likeF);
                    else
                        likeF = cl[((size_t)k*C + c)*4 + s] * bs[s] + likeF;
                    }
            likeF = likeF * (float) ev->category_weights[0];
            }
        else
            {
            likeF = 0.0f;
            for (k=0; k<K; k++)
                {
                catLike = 0.0f;
                for (s=0; s<S; s++)
                    catLike = catLike + cl[((size_t)k*C + c)*S + s] * bs[s];
                likeF = likeF + catLike * (float) ev->category_weights[k];
                }
            }
        like = (double) likeF;
        if ((ev->flags & MB200_FLAG_RANGE_GUARD) && S == 4 && likeF < 1.0e-24f)
            o->guardHit = 1;
        likeI = 0.0;
        if (ev->has_p_invar)
            {
            /* invariable-site CL = AND of the tip sets (InitInvCondLikes, src/mcmc.c:6712-6790) */
            inv = ~(uint64_t)0;
            for (t=0; t<o->cfg.tip_count; t++)
                inv &= o->tips[(size_t)t*C + c];
            if (S == 4)
                {
                likeIF = ((inv & 1) ? 1.0f : 0.0f) * bs[0];
                for (s=1; s<4; s++)
                    {
                    if (o->arith == ORC_ARITH_FMA)
                        likeIF = fmaf (((inv >> s) & 1) ? 1.0f : 0.0f, bs[s], likeIF);
                    else
                        likeIF = (((inv >> s) & 1) ? 1.0f : 0.0f) * bs[s] + likeIF;
                    }
                likeIF = likeIF * (float) ev->p_invar;
                likeI = (double) likeIF;
                }
            else
                {
                for (s=0; s<S; s++)
                    if ((inv >> s) & 1)
                        likeI += ev->state_freqs[s] * ev->p_invar;
                }
            }

        if (!ev->has_p_invar)
            {
            if (like < ORC_LIKE_EPSILON)
                { *lnL = -DBL_MAX; return MB200_EVAL_UNDERFLOW; }
            lnLike = lnScaler[c] + log (like);
            }
        else if (quirk)
            {
            if (lnScaler[c] < -200)
                {
                if (likeI > 1E-70)
                    like = likeI;
                }
            else
                like = like + (likeI / exp (lnScaler[c]));
            if (like < ORC_LIKE_EPSILON)
                { *lnL = -DBL_MAX; return MB200_EVAL_UNDERFLOW; }
            lnLike = lnScaler[c] + log (like);
            }
        else
            {
            if (lnScaler[c] < -200.0)
                {
                if (likeI > 1E-70)
                    lnLike = log (likeI);
                else
                    lnLike = log (like) + lnScaler[c];
                }
            else
                lnLike = log (like + (likeI / exp (lnScaler[c]))) + lnScaler[c];
            if (like < ORC_LIKE_EPSILON)
                { *lnL = -DBL_MAX; return MB200_EVAL_UNDERFLOW; }
            }
        sum += lnLike * w[c];
        }
    *lnL = sum;
    return MB200_EVAL_OK;
}


/* ---------------------------------------------------------------------------------------------
 * Variable-state (STANDARD data) divisions: the reference's *_Std family.  Conditional likelihoods
 * are ragged, [k][c][nStates[c]] (src/likelihood.c:1941-1943); a branch's transition matrices are
 * one block of tiProbLength floats in which pattern c's category-k matrix sits at
 * tiIndex[c] + k*nStates^2 (src/likelihood.c:1958-1961).  numBetaCats == 1 only.
 * --------------------------------------------------------------------------------------------- */
#define ORC_BRLENS_MIN ((double)0.00000001f)   /* src/bayes.h:318 */
#define ORC_BRLENS_MAX ((double)100.0f)        /* src/bayes.h:319 */

int orc_set_pattern_states (int instance, const int *ns, const int *ti, const int *bs, int matLen, int dummy, int uncompressed)
{
    int c, C;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (!o->std) return MB200_ERROR_UNSUPPORTED;
    if (!ns || !ti || !bs || matLen < 1 || dummy < 0 || dummy > o->cfg.pattern_count) return MB200_ERROR_OUT_OF_RANGE;
    C = o->cfg.pattern_count;
    for (c=0; c<C; c++)
        if (ns[c] < 2 || ns[c] > o->cfg.state_count || ti[c] < 0 || ti[c] + o->cfg.category_count * ns[c] * ns[c] > matLen ||
            bs[c] < 0 || bs[c] + ns[c] > MB200_MAX_STATES)
            return MB200_ERROR_OUT_OF_RANGE;
    free (o->nStates); free (o->tiIndex); free (o->bsIndex); free (o->clOff);
    o->nStates = (int *) malloc ((size_t)C * sizeof(int));
    o->tiIndex = (int *) malloc ((size_t)C * sizeof(int));
    o->bsIndex = (int *) malloc ((size_t)C * sizeof(int));
    o->clOff   = (size_t *) malloc ((size_t)(C + 1) * sizeof(size_t));
    memcpy (o->nStates, ns, (size_t)C * sizeof(int));
    memcpy (o->tiIndex, ti, (size_t)C * sizeof(int));
    memcpy (o->bsIndex, bs, (size_t)C * sizeof(int));
    o->clOff[0] = 0;
    for (c=0; c<C; c++)
        o->clOff[c+1] = o->clOff[c] + (size_t)ns[c];
    o->matLen = matLen; o->dummy = dummy; o->uncompressed = uncompressed;
    free (o->matrices);
    o->matrices = (float *) calloc ((size_t)o->cfg.matrix_count * (size_t)matLen, sizeof(float));
    return MB200_SUCCESS;
}

/* TiProbs_Std, equal state frequencies, unordered characters (src/likelihood.c:10066-10173): one
 * [K][n][n] run per state count n that occurs, in increasing n, which is where tiIndex points */
static void StdTiProbs (OrcInst *o, const mb200_matrix_update *mu, const mb200_evaluation *ev)
{
    int     K = o->cfg.category_count, C = o->cfg.pattern_count, c, n, k, i, j, index, found;
    double  length = mu->length, v, eV1;
    float   pNoChange, pChange, *tiP = o->matrices + (size_t)mu->matrix * o->matLen;

    if (length > ORC_BRLENS_MAX)
        length = ORC_BRLENS_MAX;
    else if (length < ORC_BRLENS_MIN)
        length = ORC_BRLENS_MIN;
    for (n=2; n<=o->cfg.state_count; n++)
        {
        found = -1;
        for (c=0; c<C && found < 0; c++)
            if (o->nStates[c] == n)
                found = o->tiIndex[c];
        if (found < 0)
            continue;                                   /* isTiNeeded[n-2] == NO */
        index = found;
        for (k=0; k<K; k++)
            {
            v = length * ev->category_rates[k];
            eV1 = exp (-((double)n / ((double)n - 1.0)) * v);
            pChange   = (float) ((1.0 / n) - ((1.0 / n) * eV1));
            pNoChange = (float) ((1.0 / n) + (((double)n - 1.0) / n) * eV1);
            if (pChange < 0.0)
                pChange = 0.0f;
            for (i=0; i<n; i++)
                for (j=0; j<n; j++)
                    tiP[index++] = (i == j) ? pNoChange : pChange;
            }
        }
}

/* one child's factor, CondLikeDown_Std / CondLikeRoot_Std inner loops (src/likelihood.c:1966-1976,
 * 4547-4559): like = sum_i P[a][i] * cl[i], accumulated from 0 with separate multiply and add */
static void StdChildTerm (OrcInst *o, int child, int matrix, float *out)
{
    int     K = o->cfg.category_count, C = o->cfg.pattern_count, c, k, a, i, n;
    size_t  numReps = o->clOff[C];
    const float *P = o->matrices + (size_t)matrix * o->matLen, *ti, *cl;
    float   x[MB200_MAX_STATES], like;
    uint64_t m;

    for (k=0; k<K; k++)
        for (c=0; c<C; c++)
            {
            n = o->nStates[c];
            if (child < o->cfg.tip_count)
                {
                /* tip conditional likelihoods: 1.0 for every state in the observed set (src/mcmc.c:6302-6330) */
                m = o->tips[(size_t)child*C + c];
                for (i=0; i<n; i++) x[i] = ((m >> i) & 1) ? 1.0f : 0.0f;
                cl = x;
                }
            else
                cl = o->partials + (size_t)(child - o->cfg.tip_count) * K * numReps + (size_t)k * numReps + o->clOff[c];
            ti = P + o->tiIndex[c] + k*n*n;
            for (a=0; a<n; a++)
                {
                like = 0.0f;
                for (i=0; i<n; i++)
                    like = like + (*ti++) * cl[i];
                out[(size_t)k * numReps + o->clOff[c] + a] = like;
                }
            }
}

static void StdOperation (OrcInst *o, const mb200_operation *op, float *lnScaler)
{
    int     K = o->cfg.category_count, C = o->cfg.pattern_count, c, k, s, n;
    size_t  numReps = o->clOff[C], tot = (size_t)K * numReps, idx;
    float  *dst = o->partials + (size_t)(op->dest - o->cfg.tip_count) * tot;
    float   scaler, *scP;

    StdChildTerm (o, op->child1, op->matrix1, o->tmp[0]);
    StdChildTerm (o, op->child2, op->matrix2, o->tmp[1]);
    if (op->child3 != MB200_NONE)
        {
        StdChildTerm (o, op->child3, op->matrix3, o->tmp[2]);
        for (idx=0; idx<tot; idx++)
            dst[idx] = o->tmp[0][idx] * o->tmp[1][idx] * o->tmp[2][idx];    /* likeL * likeR * likeA (:4559) */
        }
    else
        for (idx=0; idx<tot; idx++)
            dst[idx] = o->tmp[0][idx] * o->tmp[1][idx];                      /* likeL * likeR (:1974) */
    o->updates += (long long) K * C;

    if (op->scale_remove != MB200_NONE && lnScaler)      /* RemoveNodeScalers (src/likelihood.c:7981-8002) */
        {
        scP = o->scalers + (size_t)op->scale_remove * C;
        for (c=0; c<C; c++)
            lnScaler[c] -= scP[c];
        }
    if (op->scale_write != MB200_NONE)                   /* CondLikeScaler_Std (src/likelihood.c:5547-5610) */
        {
        scP = o->scalers + (size_t)op->scale_write * C;
        for (c=0; c<C; c++)
            {
            n = o->nStates[c];
            scaler = 0.0f;
            for (k=0; k<K; k++)
                for (s=0; s<n; s++)
                    if (dst[(size_t)k*numReps + o->clOff[c] + s] > scaler)
                        scaler = dst[(size_t)k*numReps + o->clOff[c] + s];
            for (k=0; k<K; k++)
                for (s=0; s<n; s++)
                    dst[(size_t)k*numReps + o->clOff[c] + s] /= scaler;
            scP[c] = (float) log (scaler);
            if (lnScaler)
                lnScaler[c] += scP[c];
            }
        }
}

/* Likelihood_Std, numBetaCats == 1 (src/likelihood.c:7401-7455, 7537) */
static int StdRootLikelihood (OrcInst *o, const mb200_evaluation *ev, const float *lnScaler, double *lnL)
{
    int     K = o->cfg.category_count, C = o->cfg.pattern_count, c, k, j, n;
    size_t  numReps = o->clOff[C];
    const float *cl = o->partials + (size_t)(ev->root_buffer - o->cfg.tip_count) * K * numReps;
    const float *w = o->weights + (size_t)ev->weights_row * C;
    const double *bs;
    double  catFreq = 1.0 / K, like, catLike, pUnobserved = 0.0, pObserved, sum = 0.0;

    for (c=0; c<C; c++)
        {
        n = o->nStates[c];
        bs = ev->state_freqs + o->bsIndex[c];
        like = 0.0;
        for (k=0; k<K; k++)
            {
            catLike = 0.0;
            for (j=0; j<n; j++)
                catLike += cl[(size_t)k*numReps + o->clOff[c] + j] * bs[j];
            like += catLike * catFreq;
            }
        if (c < o->dummy)
            {
            pUnobserved += like * exp (lnScaler[c]);
            continue;
            }
        if (like < ORC_LIKE_EPSILON)
            { *lnL = -DBL_MAX; return MB200_EVAL_UNDERFLOW; }
        sum += (lnScaler[c] + log (like)) * w[c];
        }
    pObserved = 1.0 - pUnobserved;
    if (pObserved < ORC_LIKE_EPSILON)
        pObserved = ORC_LIKE_EPSILON;
    sum -= log (pObserved) * (o->uncompressed);
    *lnL = sum;
    return MB200_EVAL_OK;
}

/* LaunchLogLikeForDivision (src/likelihood.c:7851-7973), one call per evaluation */
int orc_evaluate (int instance, const mb200_evaluation *evs, int count, double *lnL, int *status)
{
    int     e, i, C;
    float  *lnScaler, *zero = NULL;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    C = o->cfg.pattern_count;
    for (e=0; e<count; e++)
        {
        const mb200_evaluation *ev = &evs[e];
        if (o->std && !o->nStates)
            return MB200_ERROR_UNSUPPORTED;             /* orc_set_pattern_states first */
        for (i=0; i<ev->matrix_update_count; i++)
            {
            if (o->std) StdTiProbs (o, &ev->matrix_updates[i], ev);
            else        TiProbs (o, &ev->matrix_updates[i], ev);
            }
        /* FlipSiteScalerSpace + ResetSiteScalers | CopySiteScalers (src/likelihood.c:7885-7889) */
        if (ev->site_scaler_dst != MB200_NONE)
            {
            lnScaler = o->scalers + (size_t)ev->site_scaler_dst * C;
            if (ev->site_scaler_src == MB200_NONE)
                memset (lnScaler, 0, (size_t)C * sizeof(float));
            else if (ev->site_scaler_src != ev->site_scaler_dst)
                memcpy (lnScaler, o->scalers + (size_t)ev->site_scaler_src * C, (size_t)C * sizeof(float));
            }
        else
            {
            zero = (float *) calloc ((size_t)C, sizeof(float));
            if (ev->site_scaler_src != MB200_NONE)
                memcpy (zero, o->scalers + (size_t)ev->site_scaler_src * C, (size_t)C * sizeof(float));
            lnScaler = zero;
            }
        o->guardHit = 0;
        for (i=0; i<ev->operation_count; i++)
            {
            if (o->std) StdOperation (o, &ev->operations[i], lnScaler);
            else        Operation (o, &ev->operations[i], ev, lnScaler);
            }
        if (ev->root_buffer != MB200_NONE)
            {
            int st = o->std ? StdRootLikelihood (o, ev, lnScaler, &lnL[e]) : RootLikelihood (o, ev, lnScaler, &lnL[e]);
            if (o->guardHit && st == MB200_EVAL_OK)
                { st = MB200_EVAL_UNDERFLOW; lnL[e] = -DBL_MAX; }
            if (status) status[e] = st;
            }
        else
            {
            if (lnL) lnL[e] = 0.0;
            if (status) status[e] = MB200_EVAL_OK;
            }
        free (zero); zero = NULL;
        }
    return MB200_SUCCESS;
}

int orc_get_partials (int instance, int buffer, float *out)
{
    size_t n;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (buffer < o->cfg.tip_count || buffer >= o->cfg.partials_count) return MB200_ERROR_OUT_OF_RANGE;
    n = (size_t)o->cfg.category_count * (o->std ? o->clOff[o->cfg.pattern_count] : (size_t)o->cfg.pattern_count * o->cfg.state_count);
    memcpy (out, o->partials + (size_t)(buffer - o->cfg.tip_count) * n, n * sizeof(float));
    return MB200_SUCCESS;
}

int orc_set_partials (int instance, int buffer, const float *in)
{
    size_t n;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (buffer < o->cfg.tip_count || buffer >= o->cfg.partials_count) return MB200_ERROR_OUT_OF_RANGE;
    n = (size_t)o->cfg.category_count * (o->std ? o->clOff[o->cfg.pattern_count] : (size_t)o->cfg.pattern_count * o->cfg.state_count);
    memcpy (o->partials + (size_t)(buffer - o->cfg.tip_count) * n, in, n * sizeof(float));
    return MB200_SUCCESS;
}

int orc_get_transition_matrix (int instance, int matrix, float *out)
{
    size_t n;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (matrix < 0 || matrix >= o->cfg.matrix_count) return MB200_ERROR_OUT_OF_RANGE;
    n = o->std ? (size_t)o->matLen : (size_t)o->cfg.category_count * o->cfg.state_count * o->cfg.state_count;
    memcpy (out, o->matrices + (size_t)matrix * n, n * sizeof(float));
    return MB200_SUCCESS;
}

/* a transition-matrix buffer filled by the caller (host layout = device layout here) */
int orc_set_transition_matrix (int instance, int matrix, const float *in)
{
    size_t n;
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (matrix < 0 || matrix >= o->cfg.matrix_count || !in) return MB200_ERROR_OUT_OF_RANGE;
    n = o->std ? (size_t)o->matLen : (size_t)o->cfg.category_count * o->cfg.state_count * o->cfg.state_count;
    memcpy (o->matrices + (size_t)matrix * n, in, n * sizeof(float));
    return MB200_SUCCESS;
}

int orc_get_scalers (int instance, int scaler, float *out)
{
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (scaler < 0 || scaler >= o->cfg.scaler_count) return MB200_ERROR_OUT_OF_RANGE;
    memcpy (out, o->scalers + (size_t)scaler * o->cfg.pattern_count, (size_t)o->cfg.pattern_count * sizeof(float));
    return MB200_SUCCESS;
}

/* a node or site scaler buffer filled by the caller */
int orc_set_scalers (int instance, int scaler, const float *in)
{
    OrcInst *o = Get (instance);
    if (!o) return MB200_ERROR_BAD_INSTANCE;
    if (scaler < 0 || scaler >= o->cfg.scaler_count || !in) return MB200_ERROR_OUT_OF_RANGE;
    memcpy (o->scalers + (size_t)scaler * o->cfg.pattern_count, in, (size_t)o->cfg.pattern_count * sizeof(float));
    return MB200_SUCCESS;
}

/* CompressData's uniqueness scan (src/model.c:2618-2686): a column joins the FIRST earlier
 * column that is identical over all taxa, otherwise it becomes a new pattern; weights are
 * integer site counts (tempSitesOfPat). */
int orc_compress_patterns (const uint64_t *matrix, int n_taxa, int n_sites,
                           int *pattern_of_site, int *first_site_of_pattern, int *weights)
{
    int site, p, t, nPat = 0, same;
    for (site=0; site<n_sites; site++)
        {
        same = 0;
        for (p=0; p<nPat; p++)
            {
            same = 1;
            for (t=0; t<n_taxa; t++)
                if (matrix[(size_t)t*n_sites + site] != matrix[(size_t)t*n_sites + first_site_of_pattern[p]])
                    { same = 0; break; }
            if (same)
                break;
            }
        if (same)
            {
            weights[p]++;
            pattern_of_site[site] = p;
            }
        else
            {
            first_site_of_pattern[nPat] = site;
            weights[nPat] = 1;
            pattern_of_site[site] = nPat;
            nPat++;
            }
        }
    return nPat;
}
