/*
 * mb200_seam.c -- host-side seam between MrBayes' C code and the H100 engine.
 *
 * This translation unit is compiled TOGETHER WITH the reference's headers
 * (-I<mrbayes>/src) and linked into the reference's `mb` binary.  It
 * re-implements the accelerator entry points that the reference declares in
 * src/mbbeagle.h:13-28 (InitBeagleInstance, LaunchBEAGLELogLikeForDivision,
 * TreeTiProbs_Beagle, TreeCondLikes_Beagle_Always_Rescale,
 * TreeLikelihood_Beagle) on top of the C-ABI in include/mb200.h instead of
 * libhmsbeagle, and it follows the arithmetic rules of the BUILT-IN path
 * (src/likelihood.c:7851-7973), which is the parity target:
 *
 *   - three-neighbour update at the interior root of unrooted trees
 *     (CondLikeRoot_*, src/likelihood.c:7920-7931) instead of BEAGLE's edge
 *     likelihood (src/mbbeagle.c:1236-1274);
 *   - TIME_MIN / TIME_MAX special cases of TiProbs_Gen
 *     (src/likelihood.c:9503-9525) instead of BRLENS_MIN clamping
 *     (src/mbbeagle.c:1453-1456);
 *   - every updated non-root interior node is rescaled (rescaleFreq == 1,
 *     src/mcmc.c:6157-6164) with RemoveNodeScalers bookkeeping
 *     (src/likelihood.c:7938-7965).
 *
 * The host keeps ALL integer state: every Flip*Space call the reference makes
 * is made here too, in the same order, so ResetFlips (src/mcmc.c:15695) keeps
 * working unmodified; the engine is addressed purely by the indices valid at
 * call time.  One LogLike call == one mb200_evaluate == one fused GPU pass.
 *
 * Four ways in, one evaluation record (mb200_evaluation) and one dispatch (SeamRootAndLaunch) behind them: the
 * mbbeagle.h entry points above; MB200LaunchLogLikeForDivision / MB200LogLike (replacements for
 * LaunchLogLikeForDivision and the division loop of LogLike: all divisions of a chain in flight together); MB200Batch*
 * (chain-batched generations: all local chains of a generation in one engine call); TiProbs_B200 ... Likelihood_B200
 * (node-granular function-pointer forms driven by the reference's own LaunchLogLikeForDivision loop).  Besides them
 * the host readers installed by MB200InstallReaders.
 *
 * No reference source text is copied: only the public structs and function
 * prototypes of the reference headers are used.
 */
#include <time.h>
#include "bayes.h"
#include "likelihood.h"
#include "mbbeagle.h"
#include "mcmc.h"
#include "model.h"
#include "utils.h"

#include "mb200.h"
#include "mb200_seam.h"

/* globals of src/mcmc.c that have no extern declaration in a header */
extern int *chainId;
extern int  numLocalChains;
/* defined in src/likelihood.c:70, not declared in likelihood.h */
int UpDateCijk (int whichPart, int whichChain);
int SetNucQMatrix (MrBFlt **a, int n, int whichChain, int division, MrBFlt rateMult, MrBFlt *rA, MrBFlt *rS);   /* src/likelihood.c:8166 */
int SetProteinQMatrix (MrBFlt **a, int n, int whichChain, int division, MrBFlt rateMult);                        /* src/likelihood.c:8765 */

#define SEAM_MAX_DIVISIONS 512

/* per local chain: dynamic rescaling (MB200_RESCALE=dynamic), the rescale frequency and the run of clean evaluations;
   how many nodes the retry flipped beyond the move's own (SeamDivision.extraFlip); state[] when the chain was queued */
typedef struct { int dynFreq, dynRun, nExtraFlip, queuedState; } SeamChain;

/* one set of scratch indices of a division, what ModelInfo's *ScratchIndex fields and unscaledNodesScratch hold:
   [node] conditional likelihoods, P(t), node scalers, unscaled nodes; site scalers; eigensystem */
typedef struct { int *cl, *ti, *ns, *un; int site, cijk; } SeamScratch;

typedef struct
    {
    int                  instance;          /* engine instance, -1 = none            */
    mb200_instance_config cfg;              /* what the instance was created for     */
    unsigned long long   tipStamp;          /* checksum of the tip data and pattern weights it holds */
    const void          *parsPtr, *weightPtr; /* where that data lived on the host (cheap staleness test) */
    int                  capOps, capMats;
    mb200_operation     *ops;
    mb200_matrix_update *mats;
    mb200_evaluation     ev;                /* evaluation being assembled            */
    int                  inlineEigen;       /* nst = 1, 2: eigensystem derived per evaluation */
    double              *eigenBlock;        /* [lambda_re(4), lambda_im(4), c_ijk(64)] of the evaluation being assembled */
    /* chain-batched generations (MB200Batch*, mb200_seam.h): one queue slot per local chain, so that the
       evaluations of all chains of a generation go to the device in ONE call */
    int                  nSlots, nQueued;
    mb200_operation     *opsArena;          /* [nSlots][capOps]  */
    mb200_matrix_update *matsArena;         /* [nSlots][capMats] */
    double              *eigArena;          /* [nSlots][72]      */
    mb200_evaluation    *qEv;               /* [nSlots] evaluations queued this generation */
    int                 *qChain;            /* [nSlots] ... and their chains */
    int                  qLaunched;
    /* results of the evaluations started last (SeamStart / SeamFinish): the queue's, or in [0] a deferred single evaluation's */
    double              *qLnL;              /* [nSlots], the tail of eigArena's block */
    int                 *qStatus;           /* [nSlots], the head of the block that also holds qChain and extraFlip */
    int                  qRc, inFlight;     /* inFlight: started with evaluate_begin, evaluate_end fetches the results */
    SeamChain           *chains;            /* [nSlots] */
    int                 *extraFlip;         /* [nSlots][capOps] nodes the retry flipped beyond the move's own */
    /* per-chain scratch sets: the reference keeps ONE scratch slot per node, shared by all chains
       (src/mcmc.c:5940-5949), which is fine while a chain is accepted or rejected before the next one is
       touched; with the accept step deferred every chain needs its own.  Chain 0 keeps the reference's. */
    int                  nScratchChains, scratchNodes;
    SeamScratch         *scr;               /* [chain]; [0] unused; the four arrays of a chain are one block (cl) */
    SeamScratch          orig;              /* the reference's set while a chain's is installed */
    int                  installed;         /* chain whose set is in place, or -1 */
    int                  extraCl, extraTi, extraNs, extraEig;  /* buffers beyond the reference's own counts */
    MrBFlt             **extraCijks;        /* host eigensystem blocks appended to m->cijks for the extra slots */
    /* host readers (MB200InstallReaders): the reference's own function pointers, what the host arrays currently mirror,
       host buffers appended to m->condLikes / m->tiProbs / m->scalers for the chain-batching scratch sets */
    LikeUpFxn            refCondLikeUp;
    PrintAncStFxn        refPrintAncStates;
    PrintSiteRateFxn     refPrintSiteRates;
    int                  omegaReaders;      /* PosSelProbs / SiteOmegas wrapped (report possel / siteomega) */
    long long            evalStamp, syncedStamp;
    int                  syncedChain, syncedState, readers;
    CLFlt              **hostExtra;         /* the appended host buffers (freed by the seam) */
    int                  nHostExtra;
    int                  stdHostP;          /* STANDARD division whose P(t) the reference's TiProbs_Std builds on the host */
    int                  hostPFailed;       /* ... and one of this evaluation's matrices could not be built or shipped */
    int                  guard;             /* dynamic rescaling: the evaluation being assembled was built with a rescale frequency > 1 */
    long long            dynRetries;
    long long            clUpdates;         /* node*pattern*rate updates issued      */
    int                  pending;           /* launched by a deferred evaluation, result not yet collected */
    int                  recording, recChain, recState;   /* function-pointer forms: evaluation being recorded */
    } SeamDivision;

static SeamDivision seamDiv[SEAM_MAX_DIVISIONS];
static int          seamInitialized = NO;
/* cijk slots the device has a copy of (bit per slot).  An evaluation that reads a slot
   the device has never seen uploads it first: chains whose first evaluation ran on the
   reference's own path, or an instance that was re-created. */
static unsigned char seamCijkSeen[SEAM_MAX_DIVISIONS][(2 * MAX_CHAINS + 8) / 8 + 1];

/* bit sets (seamCijkSeen, the per-chain division flags seamFlag*) */
static inline int  SeamBitGet (const unsigned char *set, int i)         { return (set[i >> 3] >> (i & 7)) & 1; }
static inline void SeamBitAssign (unsigned char *set, int i, int on)
{
    set[i >> 3] = (unsigned char)((set[i >> 3] & ~(1 << (i & 7))) | ((on ? 1 : 0) << (i & 7)));
}

/* ---- backend indirection: lets the oracle harness record or shadow every call ---- */
static int be_create (const mb200_instance_config *c, int *i)          { return mb200_create_instance (c, i); }
static int be_finalize (int i)                                         { return mb200_finalize_instance (i); }
static int be_tips (int i, int t, const uint64_t *m)                   { return mb200_set_tip_states (i, t, m); }
static int be_weights (int i, int r, const float *w)                   { return mb200_set_pattern_weights (i, r, w); }
static int be_cijk (int i, int e, const double *b)                     { return mb200_set_cijk (i, e, b); }
static int be_eval (int i, const mb200_evaluation *e, int n, double *l, int *s) { return mb200_evaluate (i, e, n, l, s); }
static int be_begin (int i, const mb200_evaluation *e, int n)          { return mb200_evaluate_begin (i, e, n); }
static int be_end (int i, double *l, int *s)                           { return mb200_evaluate_end (i, l, s); }
static int be_pstates (int i, const int *n, const int *t, const int *b, int ml, int nd, int nu) { return mb200_set_pattern_states (i, n, t, b, ml, nd, nu); }
static int be_getp (int i, int b, float *o)                            { return mb200_get_partials (i, b, o); }
static int be_getm (int i, int m, float *o)                            { return mb200_get_transition_matrix (i, m, o); }
static int be_gets (int i, int s, float *o)                            { return mb200_get_scalers (i, s, o); }
static int be_setm (int i, int m, const float *in)                     { return mb200_set_transition_matrix (i, m, in); }
static int be_rates (int i, int e, int l, const double *q, const double *f) { return mb200_set_rate_matrices (i, e, l, q, f); }

static const MB200SeamBackend seamEngine = { be_create, be_finalize, be_tips, be_weights, be_cijk, be_eval, be_begin, be_end, be_pstates, be_getp, be_getm, be_gets, be_setm, be_rates };
static MB200SeamBackend        seamCustomBackend;           /* the table MB200SeamSetBackend was given */
static const MB200SeamBackend *seamBackend = &seamEngine;
/* what SeamRootAndLaunch does with the evaluation it has assembled: evaluate it and hand the result back; start it and
   let SeamCollect fetch the result (MB200LogLike, LaunchBEAGLELogLikeMultiPartition); keep it in the division's queue
   until MB200BatchFlush (MB200BatchQueueLogLike) */
enum { SEAM_RUN_NOW, SEAM_RUN_DEFERRED, SEAM_RUN_QUEUED };
static int seamRun = SEAM_RUN_NOW;
static int seamBatchWanted = NO;    /* MB200BatchEnable: instances are created with per-chain scratch buffers */
static void SeamScratchCounts (ModelInfo *m, int *nCl, int *nTi, int *nNs);
static int  SeamReadersWanted (ModelInfo *m);
static void SeamDropDivision (int division);

void MB200SeamSetBackend (const MB200SeamBackend *backend)
{
    if (backend == NULL)
        seamBackend = &seamEngine;
    else
        {
        seamCustomBackend = *backend;
        seamBackend = &seamCustomBackend;
        }
}

static void SeamInit (void)
{
    int d;
    if (seamInitialized == YES)
        return;
    for (d=0; d<SEAM_MAX_DIVISIONS; d++)
        {
        memset (&seamDiv[d], 0, sizeof(SeamDivision));
        seamDiv[d].instance = -1;
        seamDiv[d].installed = -1;
        }
    seamInitialized = YES;
}

/* host time spent on eigensystems (UpDateCijk: rate matrix, GetEigens, CalcCijk) and on shipping them to the engine */
static double    seamSecCijk = 0.0, seamSecCijkUpload = 0.0;
static long long seamCijkUpdates = 0;
static double SeamNow (void)
{
    struct timespec ts;
    clock_gettime (CLOCK_MONOTONIC, &ts);
    return (double) ts.tv_sec + 1e-9 * (double) ts.tv_nsec;
}
static int SeamUpDateCijk (int d, int chain)
{
    double t0 = SeamNow ();
    int    rc = UpDateCijk (d, chain);
    seamSecCijk += SeamNow () - t0;
    seamCijkUpdates++;
    return rc;
}
void MB200SeamCijkTimes (double *secHost, double *secUpload, long long *updates)
{
    if (secHost)   *secHost = seamSecCijk;
    if (secUpload) *secUpload = seamSecCijkUpload;
    if (updates)   *updates = seamCijkUpdates;
}

long long MB200SeamRescaleRetries (void)
{
    long long n = 0;
    int       d;
    if (seamInitialized == YES)
        for (d=0; d<SEAM_MAX_DIVISIONS; d++)
            n += seamDiv[d].dynRetries;
    return n;
}

long long MB200SeamUpdateCount (int division)
{
    if (seamInitialized == NO || division < 0 || division >= SEAM_MAX_DIVISIONS)
        return 0;
    return seamDiv[division].clUpdates;
}

int MB200SeamInstance (int division)
{
    if (seamInitialized == NO || division < 0 || division >= SEAM_MAX_DIVISIONS)
        return -1;
    return seamDiv[division].instance;
}

/* 4x4 nucleotide models with nst = 1 or 2 (JC69, F81, K80, HKY85): the reference evaluates
 * them with closed forms (TiProbs_JukesCantor / _Fels / _Hky, src/likelihood.c:9289, 9709, 9846)
 * and keeps no eigensystem for them in non-BEAGLE builds (InitEigenSystemInfo, src/mcmc.c:6540-6552).
 * The seam derives the eigensystem of their rate matrix for every evaluation and ships it with
 * the call (mb200_evaluation.inline_eigen), so the engine needs no extra kernel. */
int MB200SeamClosedFormModel (ModelInfo *m)
{
    if ((m->dataType == DNA || m->dataType == RNA) && m->nucModelId == NUCMODEL_4BY4 &&
        (m->nst == 1 || m->nst == 2) && m->numModelStates == 4 && m->switchRates == NULL && m->nCijkParts == 0)
        return YES;
    return NO;
}

/* Q of HKY85 (kappa = 1: F81 / JC69), scaled to one expected substitution per unit time -- the
 * same normalisation as TiProbs_Hky's beta (src/likelihood.c:9745) -- then GetEigens + CalcCijk,
 * the two public utilities UpDateCijk itself uses (src/likelihood.c:10626-10661) */
static int SeamClosedFormEigen (ModelInfo *m, int chain, double *block)
{
    int             i, j, isComplex;
    MrBFlt          kappa, *bs, scaler, mult, **q, **eigvecs, **inverseEigvecs, eigenValues[4], eigvalsImag[4];
    MrBComplex      **Ceigvecs, **CinverseEigvecs;

    bs = GetParamSubVals (m->stateFreq, chain, state[chain]);
    kappa = (m->nst == 2) ? *GetParamVals (m->tRatio, chain, state[chain]) : 1.0;
    q = AllocateSquareDoubleMatrix (4);
    eigvecs = AllocateSquareDoubleMatrix (4);
    inverseEigvecs = AllocateSquareDoubleMatrix (4);
    Ceigvecs = AllocateSquareComplexMatrix (4);
    CinverseEigvecs = AllocateSquareComplexMatrix (4);
    for (i=0; i<4; i++)
        q[i][i] = 0.0;
    scaler = 0.0;
    for (i=0; i<4; i++)
        for (j=i+1; j<4; j++)
            {
            mult = ((i == 0 && j == 2) || (i == 1 && j == 3)) ? kappa : 1.0;   /* A<->G, C<->T */
            q[i][i] -= (q[i][j] = bs[j] * mult);
            q[j][j] -= (q[j][i] = bs[i] * mult);
            scaler += bs[i] * q[i][j];
            scaler += bs[j] * q[j][i];
            }
    scaler = 1.0 / scaler;
    for (i=0; i<4; i++)
        for (j=0; j<4; j++)
            q[i][j] *= scaler;
    isComplex = GetEigens (4, q, eigenValues, eigvalsImag, eigvecs, inverseEigvecs, Ceigvecs, CinverseEigvecs);
    if (isComplex == NO)
        {
        for (i=0; i<4; i++)
            {
            block[i] = eigenValues[i];
            block[4+i] = eigvalsImag[i];
            }
        CalcCijk (4, block + 8, eigvecs, inverseEigvecs);
        }
    FreeSquareDoubleMatrix (q);
    FreeSquareDoubleMatrix (eigvecs);
    FreeSquareDoubleMatrix (inverseEigvecs);
    FreeSquareComplexMatrix (Ceigvecs);
    FreeSquareComplexMatrix (CinverseEigvecs);
    return (isComplex == NO) ? NO_ERROR : ERROR;
}

/* Codon models with omega categories (NY98, M3: lset omegavar=...): one rate matrix, hence one
 * eigensystem, per category (nCijkParts = numOmegaCats, InitEigenSystemInfo src/mcmc.c:6573-6577);
 * P(t) from TiProbs_GenCov (src/likelihood.c:9568), pruning CondLikeDown/Root/Scaler_NY98
 * (:1575, :4010, :5413), root Likelihood_NY98 (:6975): the general-S arithmetic with
 * K = numOmegaCats and the omega category frequencies as category weights. */
static int SeamOmegaCategories (ModelInfo *m)
{
    if ((m->dataType != DNA && m->dataType != RNA) || m->nucModelId != NUCMODEL_CODON)
        return NO;
    if (m->numOmegaCats <= 1 || m->numOmegaCats > MB200_MAX_CATEGORIES || m->numRateCats != 1)
        return NO;
    if (m->nCijkParts != m->numOmegaCats || m->omega == NULL || m->pInvar != NULL)
        return NO;
    return YES;
}

/* Covarion models with gamma rate variation (lset covarion=yes rates=gamma; nucleotide S = 8, protein
 * S = 40): the category's rate sits inside its own rate matrix, so there is one eigensystem per
 * rate category (nCijkParts = numRateCats, InitEigenSystemInfo src/mcmc.c:6533-6563) and P(t) comes
 * from TiProbs_GenCov; everything downstream is the general-S path (CondLike*_Gen*, Likelihood_Gen*).
 * Covarion without rate variation has nCijkParts = 1 and goes through TiProbs_Gen like any other model. */
static int SeamCovarionGamma (ModelInfo *m)
{
    if (m->switchRates == NULL || m->numOmegaCats != 1)
        return NO;
    if (m->nCijkParts <= 1 || m->nCijkParts != m->numRateCats)
        return NO;
    return YES;
}

/* one eigensystem per category? (TiProbs_GenCov models) */
static int SeamCategoryEigens (ModelInfo *m)
{
    return (SeamOmegaCategories (m) == YES || SeamCovarionGamma (m) == YES) ? YES : NO;
}

/* rate / omega categories of the division as the engine sees them */
static int SeamCategories (ModelInfo *m)
{
    return (SeamOmegaCategories (m) == YES) ? m->numOmegaCats : m->numRateCats;
}

/* STANDARD (morphological) data, the *_Std kernel family (SetLikeFunctions, src/mcmc.c:18300-18308).
 * Covered: the equal-frequency Mk model (prset symdirihyperpr=fixed(infinity): SYMPI_EQUAL) on
 * unordered characters with any number of gamma categories -- cynmix.nex's morphology partition.
 * Ordered characters, unequal state frequencies (beta categories for binary characters, one
 * eigensystem per multistate character, TiProbs_Std's second half src/likelihood.c:10410-10470) and
 * state counts whose frequency table does not fit mb200_evaluation.state_freqs stay on the
 * reference's own kernels. */
/* Who builds P(t) of a STANDARD division?  The engine, when every matrix is the equal-frequency Mk matrix of an unordered
 * character (two values per state count and category: TiProbs_Std's first loop, src/likelihood.c:10143-10173).  Ordered
 * characters (closed forms for 3 .. 6 states, :10175-10405) and unequal state frequencies (binary closed form, one
 * eigensystem per multistate character, :10410-10470) keep the reference's own TiProbs_Std: the seam calls it for every
 * dirty branch -- it writes the host array of the branch's slot -- and ships the buffer (set_transition_matrix); pruning,
 * rescaling and the root stay on the engine, which reads every entry of a caller-supplied matrix. */
static int SeamStdHostMatrices (ModelInfo *m)
{
    int c;
    if (m->dataType != STANDARD || m->stateFreq == NULL || m->cType == NULL)
        return NO;
    if (m->stateFreq->paramId != SYMPI_EQUAL)
        return YES;
    for (c=0; c<m->numChars; c++)
        if (m->cType[c] != UNORD)
            return YES;
    return NO;
}

static int SeamStdDivision (ModelInfo *m)
{
    int c, freqLen = 0;

    if (m->dataType != STANDARD)
        return NO;
    if (getenv ("MB200_NO_STD") != NULL)
        return NO;                              /* A/B switch: leave these divisions on the reference's kernels */
    if (m->stateFreq == NULL || m->numBetaCats != 1)
        return NO;
    if (m->pInvar != NULL || m->switchRates != NULL || m->numOmegaCats != 1 || m->nStates == NULL ||
        m->tiIndex == NULL || m->bsIndex == NULL || m->cType == NULL)
        return NO;
    for (c=0; c<m->numChars; c++)
        {
        if ((m->cType[c] != UNORD && m->cType[c] != ORD) || m->nStates[c] < 2 || m->nStates[c] > MB200_MAX_STATES)
            return NO;
        if (m->bsIndex[c] + m->nStates[c] > freqLen)
            freqLen = m->bsIndex[c] + m->nStates[c];
        }
    if (freqLen > MB200_MAX_STATES)
        return NO;
    if (SeamStdHostMatrices (m) == YES && seamBackend->set_transition_matrix == NULL)
        return NO;
    return YES;
}

static int SeamStdMaxStates (ModelInfo *m)
{
    int c, n = 2;
    for (c=0; c<m->numChars; c++)
        if (m->nStates[c] > n)
            n = m->nStates[c];
    return n;
}

/* ancestral states or site rates requested for the division (its CL buffers are then read on the host at sample time) */
static int SeamReadersWanted (ModelInfo *m)
{
    return (m->printAncStates == YES || m->printSiteRates == YES) ? YES : NO;
}

/* Which divisions the engine takes; everything else stays on the reference's own
 * function pointers, the way the reference keeps BEAGLE away from models it does
 * not cover (src/mcmc.c:5741-5775). */
int MB200SeamDivisionSupported (ModelInfo *m)
{
    if (m->parsModelId == YES)
        return NO;
    if (m->dataType == STANDARD)
        {
        if (SeamStdDivision (m) == NO || m->gibbsGamma == YES || m->correlation != NULL || m->nParsIntsPerSite != 1 ||
            m->numRateCats < 1 || m->numRateCats > MB200_MAX_CATEGORIES ||
            m->printAncStates == YES || m->printSiteRates == YES)
            return NO;                          /* (readers of the ragged Std buffers: not covered) */
        return YES;
        }
    if (m->dataType != DNA && m->dataType != RNA && m->dataType != PROTEIN)
        return NO;                              /* RESTRICTION / CONTINUOUS: outside the path */
    if (m->nCijkParts != 1 && MB200SeamClosedFormModel (m) == NO && SeamCategoryEigens (m) == NO)
        return NO;
    if (m->gibbsGamma == YES || m->correlation != NULL)
        return NO;
    if (m->switchRates != NULL && getenv ("MB200_NO_COVARION") != NULL)
        return NO;                              /* covarion (TiProbs_GenCov with hidden states, on/off frequencies): A/B switch.
                                                   Parity is pinned on a build of the reference WITHOUT SIMD switches
                                                   (oracle/_ref/mb_b200_scalar): the reference evaluates these models with its scalar
                                                   kernel family, which reads SIMD-laid-out buffers in an SSE-enabled build (lnL
                                                   -1558.16 on primates there, -9051.351 in the scalar build and on the engine) */
    if (m->numModelStates < 2 || m->numModelStates > MB200_MAX_STATES)
        return NO;
    if (m->numRateCats < 1 || m->numRateCats > MB200_MAX_CATEGORIES)
        return NO;
    if (m->numOmegaCats != 1 && SeamOmegaCategories (m) == NO)
        return NO;
    if (m->nParsIntsPerSite != 1)
        return NO;
    if ((m->printPosSel == YES || m->printSiteOmegas == YES) &&
        (seamBackend->get_partials == NULL || SeamOmegaCategories (m) == NO || getenv ("MB200_NO_READERS") != NULL))
        return NO;                              /* PosSelProbs / SiteOmegas read the root's conditional likelihoods on the host
                                                   (src/mcmc.c:5761-5772, 12627, 12664): MB200InstallReaders wraps them too */
    if (SeamReadersWanted (m) == YES &&
        (seamBackend->get_partials == NULL || seamBackend->get_transition_matrix == NULL || seamBackend->get_scalers == NULL ||
         m->numOmegaCats != 1 || getenv ("MB200_NO_READERS") != NULL))
        return NO;                              /* ancestral states / site rates without a read-back path */
    return YES;
}

/* Which GPU a division's buffers live on.  One process per GPU (MPI / torchrun style launch: the
 * local rank picks the device, src/mcmc.c:18331 SetLocalChainsAndDataSplits gives the process its
 * chains), or one process driving several GPUs with the partitions of every chain dealt out round
 * robin (MB200_SHARD=partitions: lnL_chain = sum over divisions, src/mcmc.c:7441, so the divisions
 * of a chain run concurrently on different devices); MB200_DEVICE pins everything to one ordinal. */
int MB200SeamDeviceFor (int division)
{
    static int  nDev = -1;
    const char *s;
    int         r = 0;

    if (nDev < 0)
        {
        nDev = mb200_device_count ();
        if (nDev < 1)
            nDev = 1;
        }
    if ((s = getenv ("MB200_DEVICE")) != NULL)
        return atoi (s);
    if ((s = getenv ("MB200_SHARD")) != NULL && strcmp (s, "partitions") == 0)
        return division % nDev;
    if ((s = getenv ("LOCAL_RANK")) != NULL || (s = getenv ("OMPI_COMM_WORLD_LOCAL_RANK")) != NULL ||
        (s = getenv ("MV2_COMM_WORLD_LOCAL_RANK")) != NULL || (s = getenv ("SLURM_LOCALID")) != NULL)
        r = atoi (s);
#   if defined (MPI_ENABLED)
    else
        r = proc_id;
#   endif
    return (r >= 0) ? r % nDev : 0;
}

/* checksum (FNV-1a) of what InitBeagleInstance uploads: tip state sets and pattern weights */
static unsigned long long SeamTipStamp (ModelInfo *m)
{
    unsigned long long  h = 1469598103934665603ULL;
    const unsigned char *b;
    size_t              i, n;
    int                 t, r;

    for (t=0; t<numLocalTaxa; t++)
        {
        b = (const unsigned char *) m->parsSets[t];
        n = (size_t) m->numChars * m->nParsIntsPerSite * sizeof(BitsLong);
        for (i=0; i<n; i++)
            h = (h ^ b[i]) * 1099511628211ULL;
        }
    for (r=0; r<chainParams.numChains; r++)
        {
        b = (const unsigned char *) (numSitesOfPat + r*numCompressedChars + m->compCharStart);
        n = (size_t) m->numChars * sizeof(CLFlt);
        for (i=0; i<n; i++)
            h = (h ^ b[i]) * 1099511628211ULL;
        }
    return h;
}

/* how many scratch slots the reference keeps per kind (entries >= 0 of its scratch index arrays) */
static void SeamScratchCounts (ModelInfo *m, int *nCl, int *nTi, int *nNs)
{
    int   i, nNodes;
    Tree *t = GetTree (m->brlens, 0, state[0]);

    nNodes = t->nNodes;
    *nCl = *nTi = *nNs = 0;
    for (i=0; i<nNodes; i++)
        {
        if (m->condLikeScratchIndex   != NULL && m->condLikeScratchIndex[i]   >= 0) (*nCl)++;
        if (m->tiProbsScratchIndex    != NULL && m->tiProbsScratchIndex[i]    >= 0) (*nTi)++;
        if (m->nodeScalerScratchIndex != NULL && m->nodeScalerScratchIndex[i] >= 0) (*nNs)++;
        }
}

/* configuration of the engine instance a division needs right now */
void MB200SeamDivisionConfig (ModelInfo *m, int division, mb200_instance_config *cfg)
{
    memset (cfg, 0, sizeof(*cfg));
    cfg->tip_count       = numLocalTaxa;
    cfg->partials_count  = m->numCondLikes;
    cfg->state_count     = (m->dataType == STANDARD) ? SeamStdMaxStates (m) : m->numModelStates;
    cfg->pattern_count   = m->numChars;
    cfg->category_count  = SeamCategories (m);
    cfg->flags           = (SeamCategoryEigens (m) == YES) ? MB200_CONFIG_CIJK_PARTS (m->nCijkParts) : 0;
    if (m->dataType == STANDARD)
        cfg->flags      |= MB200_CONFIG_VARIABLE_STATES;
    if (SeamReadersWanted (m) == YES)
        cfg->flags      |= MB200_CONFIG_SCALAR_KERNELS;     /* the reference's scalar kernel family (src/mcmc.c:17971-17992) */
    cfg->matrix_count    = m->numTiProbs;
    cfg->scaler_count    = m->numScalers;
    cfg->eigen_count     = numLocalChains + 1;    /* unused (but harmless) for the inline-eigen models */
    cfg->weight_rows     = chainParams.numChains;
    cfg->device          = MB200SeamDeviceFor (division);
    cfg->max_evaluations = (numLocalChains > 0) ? numLocalChains : 1;
    if (seamBatchWanted == YES && numLocalChains > 1)
        {
        /* chain-batched generations: every chain but the first gets scratch buffers of its own */
        int extraCl, extraTi, extraNs;
        SeamScratchCounts (m, &extraCl, &extraTi, &extraNs);
        cfg->partials_count += (numLocalChains - 1) * extraCl;
        cfg->matrix_count   += (numLocalChains - 1) * extraTi;
        cfg->scaler_count   += (numLocalChains - 1) * (extraNs + 1);   /* + the site-scaler scratch */
        cfg->eigen_count    += (numLocalChains - 1);
        }
}

/* ---- per-chain scratch sets (chain-batched generations) ------------------------------------------
 * Flip*Space (src/likelihood.c:5614-5682) swaps a chain's index with the division's ONE scratch entry;
 * installing a chain's own scratch arrays in ModelInfo before its proposal, evaluation or ResetFlips and
 * putting the reference's arrays back afterwards gives every chain a private double buffer without touching
 * any of the reference's code. */
/* puts *s into ModelInfo and returns the set that was there */
static SeamScratch SeamSwapScratch (ModelInfo *m, const SeamScratch *s)
{
    const SeamScratch was = { m->condLikeScratchIndex, m->tiProbsScratchIndex, m->nodeScalerScratchIndex, m->unscaledNodesScratch,
                              m->siteScalerScratchIndex, m->cijkScratchIndex };
    m->condLikeScratchIndex   = s->cl;
    m->tiProbsScratchIndex    = s->ti;
    m->nodeScalerScratchIndex = s->ns;
    m->unscaledNodesScratch   = s->un;
    m->siteScalerScratchIndex = s->site;
    m->cijkScratchIndex       = (s->cijk >= 0) ? s->cijk : was.cijk;    /* no cijk slot of its own: the one in place stays */
    return was;
}

static void SeamInstallScratch (ModelInfo *m, SeamDivision *sd, int chain)
{
    if (chain < 1 || chain >= sd->nScratchChains || sd->installed >= 0)
        return;
    sd->orig = SeamSwapScratch (m, &sd->scr[chain]);
    sd->installed = chain;
}

static void SeamRestoreScratch (ModelInfo *m, SeamDivision *sd)
{
    SeamScratch *mine, was;

    if (sd->installed < 0)
        return;
    mine = &sd->scr[sd->installed];
    was = SeamSwapScratch (m, &sd->orig);
    mine->site = was.site;              /* scalars travel by value; the arrays were flipped in place */
    if (mine->cijk >= 0)
        mine->cijk = was.cijk;
    sd->installed = -1;
}

/* build the scratch sets of chains 1 .. n-1: new buffer indices beyond the reference's own counts, laid out
   like the reference's scratch arrays (src/mcmc.c:5940-5949, 6139-6150, 6026-6046) */
static int SeamBuildScratchSets (ModelInfo *m, SeamDivision *sd)
{
    int   c, i, n = numLocalChains, nNodes, nextCl, nextTi, nextNs, nextEig;
    Tree *t = GetTree (m->brlens, 0, state[0]);

    nNodes = t->nNodes;
    sd->scratchNodes = nNodes;
    sd->nScratchChains = n;
    sd->scr        = (SeamScratch *) SafeCalloc ((size_t)n, sizeof(SeamScratch));
    sd->extraCijks = (MrBFlt **)     SafeCalloc ((size_t)n, sizeof(MrBFlt *));
    if (!sd->scr || !sd->extraCijks)
        return (ERROR);
    nextCl  = m->numCondLikes;
    nextTi  = m->numTiProbs;
    nextNs  = m->numScalers;
    nextEig = numLocalChains + 1;
    if (m->cijks != NULL && m->nCijkParts > 0 && m->cijkLength > 0)
        {
        /* the host computes eigensystems into m->cijks[index] (UpDateCijk): the extra slots need host blocks too */
        MrBFlt **grown = (MrBFlt **) SafeRealloc ((void *) m->cijks, (size_t)(numLocalChains + n) * sizeof(MrBFlt *));
        if (!grown)
            return (ERROR);
        m->cijks = grown;
        }
    for (c=1; c<n; c++)
        {
        SeamScratch *s = &sd->scr[c];
        s->cl = (int *) SafeMalloc ((size_t)4 * nNodes * sizeof(int));
        if (!s->cl)
            return (ERROR);
        s->ti = s->cl + nNodes;
        s->ns = s->ti + nNodes;
        s->un = s->ns + nNodes;
        for (i=0; i<nNodes; i++)
            {
            s->cl[i] = (m->condLikeScratchIndex[i]   >= 0) ? nextCl++ : -1;
            s->ti[i] = (m->tiProbsScratchIndex[i]    >= 0) ? nextTi++ : -1;
            s->ns[i] = (m->nodeScalerScratchIndex[i] >= 0) ? nextNs++ : -1;
            s->un[i] = m->unscaledNodesScratch[i];
            }
        s->site = nextNs++;
        s->cijk = -1;
        if (m->cijks != NULL && m->nCijkParts > 0 && m->cijkLength > 0)
            {
            sd->extraCijks[c] = (MrBFlt *) SafeMalloc ((size_t)m->cijkLength * sizeof(MrBFlt));
            if (!sd->extraCijks[c])
                return (ERROR);
            m->cijks[nextEig] = sd->extraCijks[c];
            s->cijk = nextEig++;
            }
        }
    return (NO_ERROR);
}

/* release everything a division holds on the engine side */
static void SeamDropDivision (int division)
{
    SeamDivision *sd = &seamDiv[division];
    int           c;

    if (sd->installed >= 0)
        SeamRestoreScratch (&modelSettings[division], sd);
    if (sd->instance >= 0)
        seamBackend->finalize_instance (sd->instance);
    free (sd->opsArena);
    free (sd->matsArena);
    free (sd->eigArena); free (sd->qStatus);    /* with qLnL; with qChain and extraFlip */
    free (sd->qEv); free (sd->chains);
    for (c=0; c<sd->nHostExtra; c++)
        free (sd->hostExtra[c]);
    free (sd->hostExtra);
    for (c=1; c<sd->nScratchChains; c++)
        {
        if (sd->scr) free (sd->scr[c].cl);
        if (sd->extraCijks) free (sd->extraCijks[c]);
        }
    free (sd->scr);
    free (sd->extraCijks);
    {
    /* the reference's reader pointers outlive the instance (the wrappers stay installed in ModelInfo) */
    const LikeUpFxn        up = sd->refCondLikeUp;
    const PrintAncStFxn    an = sd->refPrintAncStates;
    const PrintSiteRateFxn sr = sd->refPrintSiteRates;
    memset (sd, 0, sizeof(SeamDivision));
    sd->refCondLikeUp = up; sd->refPrintAncStates = an; sd->refPrintSiteRates = sr;
    }
    sd->syncedStamp = -1;
    sd->installed = -1;
    sd->instance = -1;
    memset (seamCijkSeen[division], 0, sizeof(seamCijkSeen[division]));
}

/* the evaluation being assembled writes into queue slot q */
static void SeamSelectSlot (SeamDivision *sd, int q)
{
    if (q < 0 || q >= sd->nSlots)
        q = 0;
    sd->ops        = sd->opsArena  + (size_t)q * sd->capOps;
    sd->mats       = sd->matsArena + (size_t)q * sd->capMats;
    sd->eigenBlock = sd->eigArena  + (size_t)q * 72;
}

/* Does the cached instance of a division still fit the model?  Two tests: this one runs for every evaluation, so it
   compares pointers and counts only -- another mcmc command in the same session (new model, character set or chain count)
   reallocates the reference's data and changes these; InitBeagleInstance, once per run and whenever this test answers YES,
   compares the whole configuration and a checksum of the tip data before it keeps or rebuilds the instance. */
static int SeamInstanceStale (ModelInfo *m, SeamDivision *sd)
{
    return (sd->parsPtr != (const void *) m->parsSets || sd->weightPtr != (const void *) numSitesOfPat ||
        sd->cfg.pattern_count != m->numChars || sd->cfg.category_count != SeamCategories (m) ||
        sd->cfg.partials_count != m->numCondLikes + sd->extraCl || sd->cfg.matrix_count != m->numTiProbs + sd->extraTi ||
        sd->cfg.scaler_count != m->numScalers + sd->extraNs || (m->dataType != STANDARD && sd->cfg.state_count != m->numModelStates) ||
        sd->cfg.weight_rows != chainParams.numChains || sd->cfg.eigen_count != numLocalChains + 1 + sd->extraEig) ? YES : NO;
}

/* ---- InitBeagleInstance (src/mbbeagle.c:60): allocate device buffers, load tips ---- */
int InitBeagleInstance (ModelInfo *m, int division)
{
    int                     i, c, b, nRep, rc, inst = -1, nSlots = 1;
    uint64_t               *masks = NULL, obs, full;
    mb200_instance_config   cfg;
    SeamDivision           *sd;
    mb200_operation        *ops = NULL;
    mb200_matrix_update    *mats = NULL;
    mb200_evaluation       *qEv = NULL;
    double                 *dbl = NULL;     /* eigArena [nSlots][72], qLnL [nSlots] */
    int                    *ints = NULL;    /* qStatus [nSlots], qChain [nSlots], extraFlip [nSlots][capOps] */
    SeamChain              *chains = NULL;

    SeamInit ();
    if (division < 0 || division >= SEAM_MAX_DIVISIONS)
        return (ERROR);
    sd = &seamDiv[division];
    if (MB200SeamDivisionSupported (m) == NO)
        return (ERROR);
    MB200SeamDivisionConfig (m, division, &cfg);
    if (sd->instance >= 0)
        {
        /* a second mcmc in the same session after lset / charset / mcmcp changes: the cached instance
           must match the model of THIS run, or it is rebuilt (the reference refuses a second run with
           BEAGLE, src/mbbeagle.c:66-69; here it simply works) */
        if (memcmp (&cfg, &sd->cfg, sizeof(cfg)) == 0 && sd->tipStamp == SeamTipStamp (m))
            {
            sd->parsPtr   = (const void *) m->parsSets;
            sd->weightPtr = (const void *) numSitesOfPat;
            return (NO_ERROR);
            }
        SeamDropDivision (division);
        }

    /* everything that can fail on the host is allocated before the instance is published: one queue slot
       (operation list, matrix list, inline eigensystem) per local chain */
    nSlots = (numLocalChains > 0) ? numLocalChains : 1;
    ops   = (mb200_operation *)     SafeCalloc ((size_t)nSlots * m->numCondLikes, sizeof(mb200_operation));
    mats  = (mb200_matrix_update *) SafeCalloc ((size_t)nSlots * m->numTiProbs,  sizeof(mb200_matrix_update));
    qEv   = (mb200_evaluation *)    SafeCalloc ((size_t)nSlots, sizeof(mb200_evaluation));
    dbl   = (double *)              SafeCalloc ((size_t)nSlots * (72 + 1), sizeof(double));
    ints  = (int *)                 SafeCalloc ((size_t)nSlots * (2 + m->numCondLikes), sizeof(int));
    chains = (SeamChain *)          SafeCalloc ((size_t)nSlots, sizeof(SeamChain));
    masks = (uint64_t *)            SafeMalloc ((size_t)m->numChars * sizeof(uint64_t));
    if (!ops || !mats || !qEv || !dbl || !ints || !chains || !masks)
        goto fail;
    for (i=0; i<nSlots; i++)
        chains[i].dynFreq = 1;

    rc = seamBackend->create_instance (&cfg, &inst);
    if (rc != MB200_SUCCESS)
        {
        MrBayesPrint ("%s   H100 engine: cannot create instance for division %d (%s)\n", spacer, division+1, mb200_error_string (rc));
        inst = -1;
        goto fail;
        }

    if (m->dataType == STANDARD)
        {
        if (seamBackend->set_pattern_states == NULL ||
            seamBackend->set_pattern_states (inst, m->nStates, m->tiIndex, m->bsIndex, m->tiProbLength,
                                            m->numDummyChars, m->numUncompressedChars) != MB200_SUCCESS)
            goto fail;
        }

    /* tip state sets: one bit per model state, hidden-state blocks replicated */
    nRep = (m->dataType == STANDARD) ? 1 : m->numModelStates / m->numStates;
    full = (m->numStates == 64) ? ~(uint64_t)0 : (((uint64_t)1 << m->numStates) - 1);
    for (i=0; i<numLocalTaxa; i++)
        {
        for (c=0; c<m->numChars; c++)
            {
            if (m->dataType == STANDARD)
                full = ((uint64_t)1 << m->nStates[c]) - 1;      /* the pattern's own states (src/mcmc.c:6316-6322) */
            obs = (uint64_t) m->parsSets[i][c * m->nParsIntsPerSite] & full;
            masks[c] = 0;
            for (b=0; b<nRep; b++)
                masks[c] |= obs << (b * m->numStates);
            if (m->dataType == STANDARD)
                masks[c] = obs;
            }
        if (seamBackend->set_tip_states (inst, i, masks) != MB200_SUCCESS)
            goto fail;
        }

    /* pattern weights, one row per heat-ordered chain id (src/likelihood.c:5830) */
    for (i=0; i<chainParams.numChains; i++)
        {
        if (seamBackend->set_pattern_weights (inst, i, numSitesOfPat + i*numCompressedChars + m->compCharStart) != MB200_SUCCESS)
            goto fail;
        }
    free (masks);

    sd->instance = inst;
    sd->cfg      = cfg;
    sd->tipStamp = SeamTipStamp (m);
    sd->parsPtr  = (const void *) m->parsSets;
    sd->weightPtr = (const void *) numSitesOfPat;
    sd->capOps   = m->numCondLikes;
    sd->capMats  = m->numTiProbs;
    sd->nSlots   = nSlots;
    sd->opsArena = ops;   sd->matsArena = mats;  sd->qEv = qEv;  sd->chains = chains;
    sd->eigArena = dbl;   sd->qLnL = dbl + (size_t)nSlots * 72;
    sd->qStatus  = ints;  sd->qChain = ints + nSlots;  sd->extraFlip = ints + 2 * nSlots;
    sd->nQueued  = 0;
    SeamSelectSlot (sd, 0);
    memset (seamCijkSeen[division], 0, sizeof(seamCijkSeen[division]));
    sd->extraCl = cfg.partials_count - m->numCondLikes;
    sd->extraTi = cfg.matrix_count - m->numTiProbs;
    sd->extraNs = cfg.scaler_count - m->numScalers;
    sd->extraEig = cfg.eigen_count - (numLocalChains + 1);
    sd->stdHostP = SeamStdHostMatrices (m);
    sd->hostPFailed = NO;
    if (seamBatchWanted == YES && numLocalChains > 1 && SeamBuildScratchSets (m, sd) == ERROR)
        {
        MrBayesPrint ("%s   H100 engine: cannot build the per-chain scratch sets of division %d\n", spacer, division+1);
        SeamDropDivision (division);
        return (ERROR);
        }

    MrBayesPrint ("%s   Using H100 engine (%s) for division %d on device %d: %d patterns x %d categories x %d states\n",
                  spacer, mb200_version_string (), division+1, cfg.device, m->numChars, SeamCategories (m), m->numModelStates);
    return (NO_ERROR);

fail:
    if (inst >= 0)
        seamBackend->finalize_instance (inst);
    free (ops); free (mats); free (qEv); free (dbl); free (ints); free (chains);
    free (masks);
    sd->instance = -1;
    return (ERROR);
}

void MB200SeamFinalize (void)
{
    int d;
    if (seamInitialized == NO)
        return;
    for (d=0; d<SEAM_MAX_DIVISIONS; d++)
        {
        SeamDropDivision (d);
        }
}

/* branch length seen by the substitution model (src/likelihood.c:9471-9496) */
static MrBFlt SeamBranchLength (ModelInfo *m, TreeNode *p, int chain)
{
    if (m->cppEvents != NULL)
        return GetParamSubVals (m->cppEvents, chain, state[chain])[p->index];
    else if (m->tk02BranchRates != NULL)
        return GetParamSubVals (m->tk02BranchRates, chain, state[chain])[p->index];
    else if (m->wnBranchRates != NULL)
        return GetParamSubVals (m->wnBranchRates, chain, state[chain])[p->index];
    else if (m->ilnBranchRates != NULL)
        return GetParamSubVals (m->ilnBranchRates, chain, state[chain])[p->index];
    else if (m->igrBranchRates != NULL)
        return GetParamSubVals (m->igrBranchRates, chain, state[chain])[p->index];
    else if (m->mixedBrchRates != NULL)
        return GetParamSubVals (m->mixedBrchRates, chain, state[chain])[p->index];
    return p->length;
}

static int SeamHostBuffersFor (ModelInfo *m, SeamDivision *sd);

/* this move cannot be evaluated: the signalling of Likelihood_* (src/likelihood.c:5857-5859); returns ERROR */
static int SeamFailMove (MrBFlt *lnL)
{
    (*lnL) = MRBFLT_NEG_MAX;
    abortMove = YES;
    return (ERROR);
}

/* P(t) of the branch above p (its slot is flipped already): one more matrix-update record of the evaluation being
   assembled -- or, in a stdHostP division, the matrix itself: the reference's TiProbs_Std fills the slot's host array and
   the engine gets a copy */
static int SeamMatrixRecord (ModelInfo *m, SeamDivision *sd, TreeNode *p, int chain)
{
    const int            idx = m->tiProbsIndex[chain][p->index];
    mb200_matrix_update *u;

    if (sd->stdHostP == YES)
        {
        return (TiProbs_Std (p, (int)(m - modelSettings), chain) == ERROR ||
                seamBackend->set_transition_matrix (sd->instance, idx, m->tiProbs[idx]) != MB200_SUCCESS) ? ERROR : NO_ERROR;
        }
    u = &sd->mats[sd->ev.matrix_update_count++];
    u->matrix = idx;
    u->eigen  = (sd->inlineEigen == YES) ? MB200_EIGEN_INLINE : (m->dataType == STANDARD) ? MB200_NONE : m->cijkIndex[chain];
    u->length = SeamBranchLength (m, p, chain);
    return (NO_ERROR);
}

static void SeamQueueMatrix (SeamDivision *sd, ModelInfo *m, TreeNode *p, int chain)
{
    FlipTiProbsSpace (m, chain, p->index);
    /* (a chain-batched run gave the chains slots beyond the reference's own table: SeamHostBuffersFor appends host
       arrays for them before TiProbs_Std writes one) */
    if ((sd->stdHostP == YES && SeamHostBuffersFor (m, sd) == ERROR) || SeamMatrixRecord (m, sd, p, chain) == ERROR)
        sd->hostPFailed = YES;
}

/* rate multipliers of TiProbs_Gen (src/likelihood.c:9432-9464): r_k = baseRate / (1 - pInvar) * catRate_k * corr */
static void SeamCategoryRates (ModelInfo *m, SeamDivision *sd, int division, int chain)
{
    int     k;
    MrBFlt  baseRate, corr, theRate, *catRate, pInvar;

    corr = 1.0;
    if (m->dataType == DNA || m->dataType == RNA)
        {
        if (m->nucModelId == NUCMODEL_DOUBLET)
            corr = 2.0;
        else if (m->nucModelId == NUCMODEL_CODON)
            corr = 3.0;
        }
    baseRate = GetRate (division, chain);
    pInvar = 0.0;
    if (m->pInvar != NULL)
        {
        pInvar = *GetParamVals (m->pInvar, chain, state[chain]);
        baseRate /= (1.0 - pInvar);
        }
    theRate = 1.0;
    if (m->shape != NULL)
        catRate = GetParamSubVals (m->shape, chain, state[chain]);
    else if (m->mixtureRates != NULL)
        catRate = GetParamSubVals (m->mixtureRates, chain, state[chain]);
    else
        catRate = &theRate;
    for (k=0; k<m->numRateCats; k++)
        sd->ev.category_rates[k] = baseRate * catRate[k] * corr;
    if (SeamCategoryEigens (m) == YES)
        for (k=0; k<SeamCategories (m); k++)
            sd->ev.category_rates[k] = corr;    /* TiProbs_GenCov: t = length * correctionFactor, nothing else */
}

/* ---- TreeTiProbs_Beagle (src/mbbeagle.c:1368): which P(t) must be rebuilt ---------- */
int TreeTiProbs_Beagle (Tree *t, int division, int chain)
{
    int             i;
    TreeNode       *p;
    ModelInfo      *m;
    SeamDivision   *sd;

    m  = &modelSettings[division];
    sd = &seamDiv[division];
    sd->ev.matrix_update_count = 0;
    sd->ev.matrix_updates      = sd->mats;

    /* same visiting order and the same flips as src/likelihood.c:7892-7918 */
    for (i=0; i<t->nIntNodes; i++)
        {
        p = t->intDownPass[i];
        if (p->left->upDateTi == YES)
            SeamQueueMatrix (sd, m, p->left, chain);
        if (p->right->upDateTi == YES)
            SeamQueueMatrix (sd, m, p->right, chain);
        if (t->isRooted == NO && p->anc->anc == NULL)
            SeamQueueMatrix (sd, m, p, chain);      /* interior root's branch: always rebuilt */
        }

    SeamCategoryRates (m, sd, division, chain);

    return (NO_ERROR);
}

/* ---- the op list: TreeCondLikes_Beagle_Always_Rescale / _No_Rescale / _Rescale_All (src/mbbeagle.c:995, 783, 884) ----
 * SEAM_OPS_POLICY   the built-in path's bookkeeping (src/likelihood.c:7938-7965): an updated node is rescaled when
 *                   unscaledNodes reaches m->rescaleFreq[chain] -- every node with the reference's rescaleFreq of 1
 *                   (src/mcmc.c:6157-6164), every few levels under the dynamic scheme below;
 * SEAM_OPS_NONE     the same updates, no node is rescaled (the first attempt of BEAGLE's dynamic scheme);
 * SEAM_OPS_ALL      EVERY interior node is recomputed and the site scalers are rebuilt from nothing (the retry after a
 *                   numerical failure).  Nodes the failed attempt has already flipped keep their slots; the others are
 *                   flipped now and RECORDED (not flagged: the tree's update flags are shared by every division that
 *                   uses it, and ResetFlips, src/mcmc.c:15695, reads them for all of them): should the move be rejected,
 *                   MB200BatchLeaveChain flips them back. */
enum { SEAM_OPS_POLICY, SEAM_OPS_NONE, SEAM_OPS_ALL };

/* destination, children and matrices of the update of node p, from the index tables as they stand (the caller has flipped
   the node's conditional-likelihood space); isRoot: the three-neighbour update of CondLikeRoot_* */
static void SeamOpRecord (ModelInfo *m, SeamDivision *sd, mb200_operation *op, TreeNode *p, int chain, int isRoot)
{
    op->dest    = m->condLikeIndex[chain][p->index];
    op->child1  = m->condLikeIndex[chain][p->left->index];
    op->matrix1 = m->tiProbsIndex [chain][p->left->index];
    op->child2  = m->condLikeIndex[chain][p->right->index];
    op->matrix2 = m->tiProbsIndex [chain][p->right->index];
    op->child3  = (isRoot == YES) ? m->condLikeIndex[chain][p->anc->index] : MB200_NONE;
    op->matrix3 = (isRoot == YES) ? m->tiProbsIndex [chain][p->index]      : MB200_NONE;
    sd->clUpdates += (long long) m->numChars * SeamCategories (m);
}

/* scaler bookkeeping of src/likelihood.c:7938-7965: the node's old scaler leaves the site scalers when the node was
   rescaled and the site scalers were copied, not reset; read BEFORE the node-scaler space is flipped */
static int SeamScaleRemove (ModelInfo *m, TreeNode *p, int chain)
{
    return (m->unscaledNodes[chain][p->index] == 0 && m->upDateAll == NO) ? m->nodeScalerIndex[chain][p->index] : MB200_NONE;
}

static int SeamBuildOps (Tree *t, int division, int chain, int mode)
{
    int                 i;
    TreeNode           *p;
    ModelInfo          *m;
    SeamDivision       *sd;
    mb200_operation    *op;

    m  = &modelSettings[division];
    sd = &seamDiv[division];
    sd->ev.operation_count = 0;
    sd->ev.operations      = sd->ops;

    for (i=0; i<t->nIntNodes; i++)
        {
        p = t->intDownPass[i];
        if (p->upDateCl != YES && mode != SEAM_OPS_ALL)
            continue;

        op = &sd->ops[sd->ev.operation_count++];

        if (mode == SEAM_OPS_ALL)
            {
            if (p->upDateCl != YES)
                {
                FlipCondLikeSpace (m, chain, p->index);
                FlipNodeScalerSpace (m, chain, p->index);
                sd->extraFlip[(size_t)chain * sd->capOps + sd->chains[chain].nExtraFlip++] = p->index;
                }
            }
        else
            {
            /* CondLikeDown_* / CondLikeRoot_* flip first, then read the child indices
               (src/likelihood.c:795-804) */
            FlipCondLikeSpace (m, chain, p->index);
            }
        SeamOpRecord (m, sd, op, p, chain, (t->isRooted == NO && p->anc->anc == NULL) ? YES : NO);

        if (mode == SEAM_OPS_ALL)
            op->scale_remove = MB200_NONE;              /* the site scalers start from zero */
        else
            {
            op->scale_remove = SeamScaleRemove (m, p, chain);
            FlipNodeScalerSpace (m, chain, p->index);
            }
        m->unscaledNodes[chain][p->index] = 1 + m->unscaledNodes[chain][p->left->index]
                                              + m->unscaledNodes[chain][p->right->index];
        if (mode != SEAM_OPS_NONE && m->unscaledNodes[chain][p->index] >= m->rescaleFreq[chain] && p->anc->anc != NULL)
            {
            op->scale_write = m->nodeScalerIndex[chain][p->index];
            m->unscaledNodes[chain][p->index] = 0;
            }
        else
            op->scale_write = MB200_NONE;
        }

    return (NO_ERROR);
}

/* the same with the chain's rescale frequency set to freq for the duration of the call: the reference's bookkeeping
   field steers the policy (m->rescaleFreq is 1 in builds without BEAGLE, src/mcmc.c:6157-6164) */
static void SeamBuildOpsAtFrequency (Tree *t, int division, int chain, int mode, int freq)
{
    ModelInfo *m = &modelSettings[division];
    const int  savedFreq = m->rescaleFreq[chain];

    m->rescaleFreq[chain] = freq;
    SeamBuildOps (t, division, chain, mode);
    m->rescaleFreq[chain] = savedFreq;
}

int TreeCondLikes_Beagle_Always_Rescale (Tree *t, int division, int chain)
{
    return SeamBuildOps (t, division, chain, SEAM_OPS_POLICY);
}

int TreeCondLikes_Beagle_No_Rescale (Tree *t, int division, int chain)
{
    return SeamBuildOps (t, division, chain, SEAM_OPS_NONE);
}

int TreeCondLikes_Beagle_Rescale_All (Tree *t, int division, int chain)
{
    return SeamBuildOps (t, division, chain, SEAM_OPS_ALL);
}

/* ---- dynamic rescaling (SURVEY 8f2; the reference's BEAGLE path has it as MB_BEAGLE_SCALE_DYNAMIC, src/mbbeagle.c:429-534,
 *      TODO:19-33 "rescaling takes a surprisingly large amount of time") -- opt-in: MB200_RESCALE=dynamic.
 * The built-in path rescales every updated node; most of those divisions and logarithms are not needed to stay inside
 * the float range.  Under the dynamic scheme a chain's nodes are rescaled when unscaledNodes reaches the chain's
 * rescale frequency f (>= 1): f grows by one after a run of clean evaluations and is halved when an evaluation
 * underflows, in which case the evaluation is REPEATED at once with every interior node recomputed and rescaled
 * (SEAM_OPS_ALL at f = 1) before the chain sees a result -- a move is never rejected because of sparse rescaling.
 * lnL then agrees with the always-rescale arithmetic to rounding (fewer divisions by the maximum; bar: 1e-6 relative),
 * which is why the default stays the reference's policy (bit-level parity). */
static int seamDynMaxFreq = 8;      /* MB200_RESCALE_MAXFREQ */
static int seamDynRun     = 200;    /* MB200_RESCALE_RUN: clean evaluations before the frequency grows */
static int seamDynForceRetry = NO;  /* MB200_RESCALE_FORCE_RETRY=1 (tests): every evaluation takes the retry path */
static int seamDynDebug   = NO;     /* MB200_RESCALE_DEBUG: one line on stderr per retry */

static int SeamDynamicRescaling (void)
{
    static int mode = -1;
    if (mode < 0)
        {
        const char *s = getenv ("MB200_RESCALE");
        mode = (s != NULL && strcmp (s, "dynamic") == 0) ? YES : NO;
        if ((s = getenv ("MB200_RESCALE_MAXFREQ")) != NULL && atoi (s) >= 1) seamDynMaxFreq = atoi (s);
        if ((s = getenv ("MB200_RESCALE_RUN")) != NULL && atoi (s) >= 1)     seamDynRun = atoi (s);
        seamDynForceRetry = (getenv ("MB200_RESCALE_FORCE_RETRY") != NULL) ? YES : NO;
        seamDynDebug      = (getenv ("MB200_RESCALE_DEBUG") != NULL) ? YES : NO;
        }
    return mode;
}

/* site scalers of the evaluation being assembled: the caller has flipped the site-scaler space; the reset or the copy
   from the scratch slot (src/likelihood.c:7885-7889) happens on the device as part of the fused pass */
static void SeamSiteScalers (ModelInfo *m, SeamDivision *sd, int chain)
{
    sd->ev.site_scaler_dst = m->siteScalerIndex[chain];
    sd->ev.site_scaler_src = (m->upDateAll == YES) ? MB200_NONE : m->siteScalerScratchIndex;
}

static int SeamApplyResult (int division, int chain, int rc, double value, int status, MrBFlt *lnL);
static int SeamRootAndLaunch (int division, int chain, int rootNode, MrBFlt *lnL, int whichSitePats);

/* Start n evaluations of a division / finish them: return code in sd->qRc, results in sd->qLnL and sd->qStatus.  With
   evaluate_begin / evaluate_end the device works between the two calls; a backend without the pair evaluates in SeamStart. */
static void SeamStart (SeamDivision *sd, const mb200_evaluation *ev, int n)
{
    sd->inFlight = (seamBackend->evaluate_begin != NULL && seamBackend->evaluate_end != NULL) ? YES : NO;
    sd->qRc = (sd->inFlight == YES) ? seamBackend->evaluate_begin (sd->instance, ev, n)
                                    : seamBackend->evaluate (sd->instance, ev, n, sd->qLnL, sd->qStatus);
}

static void SeamFinish (SeamDivision *sd)
{
    if (sd->inFlight == YES && sd->qRc == MB200_SUCCESS)
        sd->qRc = seamBackend->evaluate_end (sd->instance, sd->qLnL, sd->qStatus);
    sd->inFlight = NO;
}

/* ---- TreeLikelihood_Beagle (src/mbbeagle.c:1117): root integration; launches ------- */
int TreeLikelihood_Beagle (Tree *t, int division, int chain, MrBFlt *lnL, int whichSitePats)
{
    return SeamRootAndLaunch (division, chain, t->root->left->index, lnL, whichSitePats);
}

/* root integration parameters of Likelihood_* (src/likelihood.c:5764-7130), then the launch */
static int SeamRootAndLaunch (int division, int chain, int rootNode, MrBFlt *lnL, int whichSitePats)
{
    int             k, s, status, rc;
    MrBFlt          pInvar, freq, *bs;
    double          value;
    ModelInfo      *m;
    SeamDivision   *sd;

    m  = &modelSettings[division];
    sd = &seamDiv[division];

    if (sd->hostPFailed == YES)
        {
        sd->hostPFailed = NO;
        return SeamFailMove (lnL);
        }
    sd->evalStamp++;
    sd->ev.root_buffer = m->condLikeIndex[chain][rootNode];
    sd->ev.weights_row = whichSitePats;
    sd->ev.flags       = 0;
    sd->ev.inline_eigen = (sd->inlineEigen == YES) ? sd->eigenBlock : NULL;

    pInvar = 0.0;
    sd->ev.has_p_invar = NO;
    if (m->pInvar != NULL)
        {
        pInvar = *GetParamVals (m->pInvar, chain, state[chain]);
        sd->ev.has_p_invar = YES;
        }
    sd->ev.p_invar = pInvar;
    /* which reference kernel family this division would run (SetLikeFunctions,
       src/mcmc.c:17995-18010 vs 18109-18243) decides two rounding-level details */
    if (m->dataType == STANDARD)
        sd->ev.flags = 0;                               /* *_Std family: dense tips, no pInvar */
    else if (m->numModelStates == 4 && (m->dataType == DNA || m->dataType == RNA))
        {
        sd->ev.flags |= MB200_FLAG_NUC4_PINVAR_QUIRK;   /* Likelihood_NUC4_* family */
        if (SeamReadersWanted (m) == YES)
            sd->ev.flags |= MB200_FLAG_TIP_SHORTCUTS;   /* scalar CondLikeDown_NUC4: preLike shortcuts (src/likelihood.c:816-832) */
        if (sd->guard == YES)
            sd->ev.flags |= MB200_FLAG_RANGE_GUARD;     /* sparsely rescaled evaluation (dynamic scheme) */
        }
    else
        sd->ev.flags |= MB200_FLAG_TIP_SHORTCUTS;       /* *_Gen_SSE family */

    /* category weights (src/likelihood.c:5821-5824) */
    if (m->pInvar == NULL)
        freq = 1.0 / m->numRateCats;
    else
        freq = (1.0 - pInvar) / m->numRateCats;
    for (k=0; k<m->numRateCats; k++)
        sd->ev.category_weights[k] = freq;
    if (SeamOmegaCategories (m) == YES)
        {
        /* Likelihood_NY98 (src/likelihood.c:6998): the omega category frequencies */
        MrBFlt *omegaCatFreq = GetParamSubVals (m->omega, chain, state[chain]);
        for (k=0; k<m->numOmegaCats; k++)
            sd->ev.category_weights[k] = omegaCatFreq[k];
        }

    if (m->dataType == STANDARD)
        {
        /* Likelihood_Std: bs = GetParamStdStateFreqs (...) + m->bsIndex[c] (src/likelihood.c:7387, 7409) */
        int c, freqLen = 0;
        for (c=0; c<m->numChars; c++)
            if (m->bsIndex[c] + m->nStates[c] > freqLen)
                freqLen = m->bsIndex[c] + m->nStates[c];
        bs = GetParamStdStateFreqs (m->stateFreq, chain, state[chain]);
        for (s=0; s<freqLen && s<MB200_MAX_STATES; s++)
            sd->ev.state_freqs[s] = bs[s];
        }
    else
        {
        bs = GetParamSubVals (m->stateFreq, chain, state[chain]);
        for (s=0; s<m->numModelStates; s++)
            sd->ev.state_freqs[s] = bs[s];
        }
    if (m->switchRates != NULL)
        {
        /* covarion: stationary frequencies of the on / off copies of every state, on-states first
           (Likelihood_Gen, src/likelihood.c:5799-5818) */
        MrBFlt *swr = GetParamVals (m->switchRates, chain, state[chain]);
        MrBFlt  probOn = swr[0] / (swr[0] + swr[1]), probOff = 1.0 - probOn;
        int     half = m->numModelStates / 2;
        for (s=0; s<half; s++)
            {
            sd->ev.state_freqs[s]        = bs[s] * probOn;
            sd->ev.state_freqs[s + half] = bs[s] * probOff;
            }
        }

    if (seamRun == SEAM_RUN_QUEUED)
        {
        /* chain-batched generation: the evaluation waits in the division's queue until MB200BatchFlush
           sends every chain's evaluation to the device in one call */
        int q = sd->nQueued;
        if (q >= sd->nSlots)
            return SeamFailMove (lnL);
        sd->qEv[q]    = sd->ev;
        sd->qChain[q] = chain;
        sd->chains[chain].queuedState = state[chain];
        sd->chains[chain].nExtraFlip  = 0;
        sd->nQueued   = q + 1;
        SeamSelectSlot (sd, q + 1);
        return (NO_ERROR);
        }
    if (seamRun == SEAM_RUN_DEFERRED)
        {
        /* partition-batched evaluation: launch only, SeamCollect fetches the result */
        SeamStart (sd, &sd->ev, 1);
        sd->pending = YES;
        return (NO_ERROR);
        }
    rc = seamBackend->evaluate (sd->instance, &sd->ev, 1, &value, &status);
    return SeamApplyResult (division, chain, rc, value, status, lnL);
}

/* dynamic rescaling, the retry: the evaluation underflowed with sparse rescaling -> every interior node of the chain's
   tree again, rescaled at every node, site scalers from zero (the P(t) of this evaluation are on the device already) */
static int SeamRetryRescaleAll (int division, int chain, double *value, int *status)
{
    ModelInfo    *m  = &modelSettings[division];
    SeamDivision *sd = &seamDiv[division];
    Tree         *t  = GetTree (m->brlens, chain, state[chain]);
    int           rc;

    if (sd->nQueued > 0 && sd->qLaunched == YES)
        {
        /* chain-batched generation: the failed evaluation is the chain's queue entry */
        int q;
        for (q=0; q<sd->nQueued; q++)
            if (sd->qChain[q] == chain)
                break;
        if (q == sd->nQueued)
            return (ERROR);
        sd->ev = sd->qEv[q];
        SeamSelectSlot (sd, q);
        }
    /* root, weights row, rates, frequencies, pInvar of the failed evaluation stay; the operations are built anew */
    SeamBuildOpsAtFrequency (t, division, chain, SEAM_OPS_ALL, 1);
    sd->ev.matrix_update_count = 0;
    sd->ev.site_scaler_dst = m->siteScalerIndex[chain];
    sd->ev.site_scaler_src = MB200_NONE;
    sd->ev.flags &= ~MB200_FLAG_RANGE_GUARD;            /* every node rescaled: only a dead likelihood fails now */
    sd->dynRetries++;
    rc = seamBackend->evaluate (sd->instance, &sd->ev, 1, value, status);
    return (rc == MB200_SUCCESS) ? NO_ERROR : ERROR;
}

/* result of an evaluation -> the reference's conventions */
static int SeamApplyResult (int division, int chain, int rc, double value, int status, MrBFlt *lnL)
{
    SeamDivision *sd = &seamDiv[division];

    if (rc == MB200_SUCCESS && SeamDynamicRescaling () == YES && chain >= 0 && chain < sd->nSlots)
        {
        SeamChain *ch = &sd->chains[chain];
        if (sd->qLaunched == YES && sd->nQueued > 0 &&
            ((status == MB200_EVAL_UNDERFLOW && ch->dynFreq > 1) || (seamDynForceRetry == YES && status == MB200_EVAL_OK)))
            {
            const double failedValue = value;
            const int    failedFreq = ch->dynFreq;
            ch->dynFreq = (ch->dynFreq + 1) / 2;
            ch->dynRun  = 0;
            if (SeamRetryRescaleAll (division, chain, &value, &status) == ERROR)
                rc = MB200_ERROR_GENERAL;
            if (seamDynDebug == YES)
                fprintf (stderr, "mb200 rescale retry: division %d chain %d freq %d: first attempt %.10g -> %.10g (status %d)\n",
                         division + 1, chain, failedFreq, failedValue, value, status);
            }
        else if (status == MB200_EVAL_OK && modelSettings[division].numModelStates == 4 && ++ch->dynRun >= seamDynRun)
            {
            ch->dynRun = 0;
            if (ch->dynFreq < seamDynMaxFreq)
                ch->dynFreq++;
            }
        }
    if (rc != MB200_SUCCESS)
        {
        MrBayesPrint ("%s   H100 engine: evaluation failed for division %d (%s)\n", spacer, division+1, mb200_error_string (rc));
        return SeamFailMove (lnL);
        }
    if (status == MB200_EVAL_UNDERFLOW)
        return SeamFailMove (lnL);
    (*lnL) = value;
    return (NO_ERROR);
}

/* ---- LaunchBEAGLELogLikeForDivision (src/mbbeagle.c:400, ALWAYS scheme) ------------ */
void LaunchBEAGLELogLikeForDivision (int chain, int d, ModelInfo *m, Tree *tree, MrBFlt *lnL)
{
    SeamDivision *sd = &seamDiv[d];

    /* site scalers: flip, then reset or copy (src/likelihood.c:7885-7889) */
    FlipSiteScalerSpace (m, chain);
    SeamSiteScalers (m, sd, chain);

    TreeTiProbs_Beagle (tree, d, chain);
    sd->guard = NO;
    /* (only inside chain-batched generations: their hooks are what can undo a retry's extra flips after a rejection) */
    if (SeamDynamicRescaling () == YES && seamRun == SEAM_RUN_QUEUED && chain < sd->nSlots && m->numModelStates == 4 &&
        (m->dataType == DNA || m->dataType == RNA) && sd->chains[chain].dynFreq > 1)
        {
        /* 4-state divisions only (the kernels that carry the float-range guard, MB200_FLAG_RANGE_GUARD): the built-in
           path's policy at the chain's own rescale frequency */
        SeamBuildOpsAtFrequency (tree, d, chain, SEAM_OPS_POLICY, sd->chains[chain].dynFreq);
        sd->guard = YES;
        }
    else
        TreeCondLikes_Beagle_Always_Rescale (tree, d, chain);
    TreeLikelihood_Beagle (tree, d, chain, lnL, chainId[chain] % chainParams.numChains);
}

/* ---- eigensystems on the device (SURVEY 8 f3; MB200_EIGEN=device|host, default: device for more than 32 states) ----
 * What UpDateCijk (src/likelihood.c:10476) does, minus GetEigens and CalcCijk: flip the cijk space, build the rate
 * matrix (or one per omega category, rescaled together so that the mean rate is one, :10676-10716) with the
 * reference's own SetNucQMatrix / SetProteinQMatrix, and hand matrices + stationary frequencies to the backend,
 * which diagonalises them on its stream while the host goes on to the next chain.  Taken only for time-reversible
 * matrices (checked here, entry by entry); anything else -- and every backend without the entry point -- keeps the
 * host path.  The host block m->cijks[idx] is NOT written on this path: nothing on the host reads it while the
 * division is on the engine (the function-pointer forms keep the host path, the reference's own driver calls
 * UpDateCijk for them). */
static MrBFlt **seamQ[SEAM_MAX_DIVISIONS][MB200_MAX_CATEGORIES];
static double  *seamQFlat[SEAM_MAX_DIVISIONS];
static int      seamQDim[SEAM_MAX_DIVISIONS], seamQParts[SEAM_MAX_DIVISIONS];   /* what the two above were allocated for */
static long long seamDeviceEigens = 0;

long long MB200SeamDeviceEigens (void) { return seamDeviceEigens; }

static int SeamDeviceEigenWanted (ModelInfo *m)
{
    /* MB200_EIGEN = device: whenever possible; host: never; unset: where it pays -- more than 32 states (codon models:
       the host's GetEigens + CalcCijk cost 1-5 ms per move there, the device 0.3-0.5 ms off the host's critical path;
       for 4 and 20 states the two are on a par) */
    static int mode = -1;
    if (mode < 0)
        {
        const char *e = getenv ("MB200_EIGEN");
        mode = (e == NULL) ? 2 : (strcmp (e, "device") == 0) ? 1 : 0;
        }
    if (mode == 0 || seamBackend->set_rate_matrices == NULL)
        return NO;
    if (mode == 2 && m->numModelStates <= 32)
        return NO;
    if (m->cijkLength <= 0 || m->switchRates != NULL || m->numModelStates > MB200_MAX_STATES)
        return NO;
    if (m->dataType == DNA || m->dataType == RNA)
        {
        if (m->nCijkParts > 1 && !(m->nucModelId == NUCMODEL_CODON && m->numOmegaCats == m->nCijkParts))
            return NO;
        return YES;
        }
    if (m->dataType == PROTEIN && m->nCijkParts == 1)
        return YES;
    return NO;
}

/* YES: the slot m->cijkIndex[chain] (after the flip) is being computed by the backend; NO: nothing was touched */
static int SeamDeviceEigen (ModelInfo *m, SeamDivision *sd, int d, int chain)
{
    const int   n = m->numModelStates, parts = (m->nCijkParts > 1) ? m->nCijkParts : 1;
    const int   codon = ((m->dataType == DNA || m->dataType == RNA) && m->nucModelId == NUCMODEL_CODON) ? YES : NO;
    int         i, j, k;
    MrBFlt      rA = 0.0, rS = 0.0, posScaler = 0.0, *omega = NULL, *omegaFreq = NULL, *bs, big = 0.0;
    double      t0 = SeamNow ();

    if (parts > MB200_MAX_CATEGORIES)
        return (NO);
    if (seamQFlat[d] != NULL && (seamQDim[d] != n || seamQParts[d] != parts))
        {
        /* another mcmc command changed the division's model: the work matrices no longer fit */
        for (k=0; k<seamQParts[d]; k++)
            { FreeSquareDoubleMatrix (seamQ[d][k]); seamQ[d][k] = NULL; }
        free (seamQFlat[d]);
        seamQFlat[d] = NULL;
        }
    if (seamQFlat[d] == NULL)
        {
        for (k=0; k<parts; k++)
            if ((seamQ[d][k] = AllocateSquareDoubleMatrix (n)) == NULL)
                return (NO);
        if ((seamQFlat[d] = (double *) SafeMalloc ((size_t) parts * n * n * sizeof(double))) == NULL)
            return (NO);
        seamQDim[d] = n; seamQParts[d] = parts;
        }
    if (codon == YES)
        {
        omega = GetParamVals (m->omega, chain, state[chain]);
        if (m->numOmegaCats > 1)
            omegaFreq = GetParamSubVals (m->omega, chain, state[chain]);
        }
    for (k=0; k<parts; k++)
        {
        if (m->dataType == PROTEIN)
            {
            if (SetProteinQMatrix (seamQ[d][k], n, chain, d, 1.0) == ERROR)
                return (NO);
            }
        else if (SetNucQMatrix (seamQ[d][k], n, chain, d, (codon == YES) ? omega[k] : 1.0, &rA, &rS) == ERROR)
            return (NO);
        if (codon == YES && m->numOmegaCats > 1)
            posScaler += omegaFreq[k] * (rS + rA);
        }
    if (codon == YES && m->numOmegaCats > 1)
        posScaler = 1.0 / posScaler;
    else
        posScaler = 1.0;
    bs = GetParamSubVals (m->stateFreq, chain, state[chain]);
    for (k=0; k<parts; k++)
        for (i=0; i<n; i++)
            for (j=0; j<n; j++)
                {
                const double q = seamQ[d][k][i][j] * posScaler;
                seamQFlat[d][((size_t) k * n + i) * n + j] = q;
                if (fabs (q) > big)
                    big = fabs (q);
                }
    /* detailed balance, entry by entry: pi_i q_ij == pi_j q_ji */
    for (i=0; i<n; i++)
        if (!(bs[i] > 0.0))
            return (NO);
    for (k=0; k<parts; k++)
        for (i=0; i<n; i++)
            for (j=i+1; j<n; j++)
                {
                const double a = bs[i] * seamQFlat[d][((size_t) k * n + i) * n + j], b = bs[j] * seamQFlat[d][((size_t) k * n + j) * n + i];
                if (fabs (a - b) > 1e-12 * big)
                    return (NO);
                }
    FlipCijkSpace (m, chain);
    /* after the flip the scratch entry is the slot of the chain's pre-proposal state: a nearby eigensystem */
    if (seamBackend->set_rate_matrices (sd->instance, m->cijkIndex[chain], m->cijkScratchIndex, seamQFlat[d], bs) != MB200_SUCCESS)
        {
        FlipCijkSpace (m, chain);       /* back; the host path flips again */
        return (NO);
        }
    SeamBitAssign (seamCijkSeen[d], m->cijkIndex[chain], YES);
    seamSecCijk += SeamNow () - t0;
    seamCijkUpdates++;
    seamDeviceEigens++;
    return (YES);
}

/* the engine's copy of the chain's eigensystem follows the host's: upload after UpDateCijk, and the
   first time a slot is read that the device has never seen */
static int SeamSyncCijk (ModelInfo *m, SeamDivision *sd, int d, int chain)
{
    int idx = m->cijkIndex[chain];

    if (idx < 0 || idx > 2 * MAX_CHAINS)
        return (ERROR);
    if (m->upDateCijk == YES || SeamBitGet (seamCijkSeen[d], idx) == 0)
        {
        double t0 = SeamNow ();
        if (seamBackend->set_cijk (sd->instance, idx, m->cijks[idx]) != MB200_SUCCESS)
            return (ERROR);
        seamSecCijkUpload += SeamNow () - t0;
        SeamBitAssign (seamCijkSeen[d], idx, YES);
        }
    return (NO_ERROR);
}

/* The model-specific part of MB200LaunchLogLikeForDivision: puts the eigensystem the evaluation reads where the engine
   looks for it (inline block, device slot, or none) and sets upDateAll like LaunchLogLikeForDivision
   (src/likelihood.c:7864-7872).  READY: launch; FAILED: the move failed, lnL (and, where the reference does, abortMove)
   are set; NOT_HANDLED: the division goes back to the reference's own path, nothing was flipped. */
enum { SEAM_EIGEN_READY, SEAM_EIGEN_FAILED, SEAM_EIGEN_NOT_HANDLED };

static int SeamPrepareEigen (ModelInfo *m, SeamDivision *sd, int d, int chain, MrBFlt *lnL)
{
    /* STANDARD data: the engine reads no eigensystem (equal-frequency Mk has none, cijkLength == 0; the others' matrices
       come from TiProbs_Std), but the reference's driver still calls UpDateCijk when flagged (src/likelihood.c:7864) -- a
       no-op for Mk -- and so does the seam; SeamDeviceEigenWanted is NO for these divisions */
    const int hasEigen = (m->dataType != STANDARD) ? YES : NO;
    int       deviceEigen = NO;

    sd->inlineEigen = MB200SeamClosedFormModel (m);
    if (sd->inlineEigen == YES)
        {
        /* no cijk bookkeeping in the reference for these models: derive the eigensystem of the
           chain's current kappa / base frequencies and send it along with the evaluation */
        if (m->upDateCijk == YES)
            m->upDateAll = YES;
        if (SeamClosedFormEigen (m, chain, sd->eigenBlock) == ERROR)
            {
            SeamFailMove (lnL);
            return SEAM_EIGEN_FAILED;
            }
        return SEAM_EIGEN_READY;
        }

    /* every reason to hand the division back to the reference's own path comes BEFORE UpDateCijk:
       that call flips the cijk space, and a second UpDateCijk by the fallback path would overwrite
       the slot ResetFlips needs to restore a rejected move (src/mcmc.c:15695) */
    if (hasEigen == YES && (m->cijkIndex[chain] < 0 || m->cijkIndex[chain] > 2 * MAX_CHAINS ||
                            m->cijkScratchIndex < 0 || m->cijkScratchIndex > 2 * MAX_CHAINS))
        return SEAM_EIGEN_NOT_HANDLED;

    if (m->upDateCijk == YES)
        {
        if (SeamDeviceEigenWanted (m) == YES && SeamDeviceEigen (m, sd, d, chain) == YES)
            deviceEigen = YES;
        else if (SeamUpDateCijk (d, chain) == ERROR)
            {
            (*lnL) = MRBFLT_NEG_MAX;        /* abortMove stays as it is: what LaunchLogLikeForDivision does (src/likelihood.c:7864-7872) */
            return SEAM_EIGEN_FAILED;
            }
        m->upDateAll = YES;
        }
    if (hasEigen == YES && deviceEigen == NO && SeamSyncCijk (m, sd, d, chain) == ERROR)
        {
        SeamFailMove (lnL);
        return SEAM_EIGEN_FAILED;
        }
    return SEAM_EIGEN_READY;
}

/* ---- replacement for LaunchLogLikeForDivision (src/likelihood.c:7851) -------------- */
/* Returns NO when the division is not handled by the engine (caller keeps the
   reference's own function-pointer path for it). */
int MB200LaunchLogLikeForDivision (int chain, int d, MrBFlt *lnL)
{
    ModelInfo    *m;
    SeamDivision *sd;
    int           eigen;

    SeamInit ();
    m = &modelSettings[d];
    if (MB200SeamDivisionSupported (m) == NO)
        return (NO);
    sd = &seamDiv[d];
    if ((sd->instance < 0 || SeamInstanceStale (m, sd) == YES) && InitBeagleInstance (m, d) == ERROR)
        return (NO);

    eigen = SeamPrepareEigen (m, sd, d, chain, lnL);
    if (eigen == SEAM_EIGEN_NOT_HANDLED)
        return (NO);
    if (eigen == SEAM_EIGEN_READY)
        LaunchBEAGLELogLikeForDivision (chain, d, m, GetTree (m->brlens, chain, state[chain]), lnL);
    return (YES);
}

/* collect the results of the deferred evaluations of the listed divisions (divisions == NULL: divisions 0 .. n-1) */
static void SeamCollect (const int *divisions, int n, int chain)
{
    int           i, d;
    SeamDivision *sd;

    for (i=0; i<n; i++)
        {
        d = (divisions != NULL) ? divisions[i] : i;
        if (d >= SEAM_MAX_DIVISIONS || seamDiv[d].pending == NO)
            continue;
        sd = &seamDiv[d];
        sd->pending = NO;
        SeamFinish (sd);
        SeamApplyResult (d, chain, sd->qRc, sd->qLnL[0], sd->qStatus[0], &(modelSettings[d].lnLike[2*chain + state[chain]]));
        }
}

/* ---- replacement for the division loop of LogLike (src/mcmc.c:7421-7441) ------------ */
MrBFlt MB200LogLike (int chain, void (*cpuPath) (int chain, int d, MrBFlt *lnL))
{
    int         d;
    ModelInfo  *m;
    MrBFlt      chainLnLike = 0.0;

    /* pass 1: launch every division that needs updating (engine) or compute it (reference path) */
    seamRun = SEAM_RUN_DEFERRED;
    for (d=0; d<numCurrentDivisions; d++)
        {
        m = &modelSettings[d];
        if (m->upDateCl != YES)
            continue;
        if (MB200LaunchLogLikeForDivision (chain, d, &(m->lnLike[2*chain + state[chain]])) == NO)
            {
            seamRun = SEAM_RUN_NOW;     /* the reference's path may reach the function-pointer forms */
            cpuPath (chain, d, &(m->lnLike[2*chain + state[chain]]));
            seamRun = SEAM_RUN_DEFERRED;
            }
        }
    seamRun = SEAM_RUN_NOW;

    /* pass 2: collect */
    SeamCollect (NULL, numCurrentDivisions, chain);
    if (abortMove == YES)
        return MRBFLT_NEG_MAX;
    for (d=0; d<numCurrentDivisions; d++)
        chainLnLike += modelSettings[d].lnLike[2*chain + state[chain]];
    return chainLnLike;
}

/* ======================================================================================
 * Chain-batched generations (SURVEY 8f1; RunChain's chain loop, src/mcmc.c:16718-16938).
 *
 * The reference proposes, evaluates and accepts or rejects one chain at a time.  Nothing in a generation couples
 * the chains except the random-number stream, so the loop can be cut in two around LogLike: phase A proposes a
 * move for EVERY local chain and queues its likelihood evaluation (all host-side work happens here, in the
 * reference's order: parameter reads, UpDateCijk, every Flip*Space), draws the chain's acceptance variate at the
 * very position of the stream where the serial loop draws it (LogLike consumes no random numbers), ONE device
 * call evaluates the generation's queue per division, and phase B applies the results chain by chain with the
 * reference's accept / reject code.  What the serial loop shares between chains and a deferred accept cannot
 * share is given per chain: the scratch index sets (SeamInstallScratch) and the division update flags that
 * ResetFlips reads (src/mcmc.c:15695-15760).
 *
 *   MB200BatchEnable (YES)            before the instances are created (they get the extra scratch buffers)
 *   MB200BatchBegin ()                start of a generation: YES when every division can be batched
 *   MB200BatchEnterChain (c, phase) / MB200BatchLeaveChain (c, phase)      bracket everything chain c does
 *   MB200BatchQueueLogLike (c)        phase A, where the serial loop calls LogLike
 *   MB200BatchFlush ()                between the phases
 *   MB200BatchFinishLogLike (c)       phase B: the chain's lnL (abortMove / MRBFLT_NEG_MAX like LogLike)
 * ====================================================================================== */
static unsigned char seamFlagCl[MAX_CHAINS][SEAM_MAX_DIVISIONS / 8], seamFlagCijk[MAX_CHAINS][SEAM_MAX_DIVISIONS / 8],
                     seamFlagAll[MAX_CHAINS][SEAM_MAX_DIVISIONS / 8];

void MB200BatchEnable (int enable)
{
    seamBatchWanted = (enable == YES) ? YES : NO;
}

int MB200BatchBegin (void)
{
    int           d;
    ModelInfo    *m;
    SeamDivision *sd;

    SeamInit ();
    if (seamBatchWanted == NO || numLocalChains < 2 || numLocalChains > MAX_CHAINS || numCurrentDivisions > SEAM_MAX_DIVISIONS ||
        chainParams.runWithData == NO)
        return (NO);
    for (d=0; d<numCurrentDivisions; d++)
        {
        m  = &modelSettings[d];
        sd = &seamDiv[d];
        /* a division on the reference's own kernels shares ITS scratch buffers between the chains: no deferral */
        if (MB200SeamDivisionSupported (m) == NO)
            return (NO);
        if (sd->instance < 0 && InitBeagleInstance (m, d) == ERROR)
            return (NO);
        if (sd->nScratchChains != numLocalChains)
            return (NO);
        sd->nQueued = 0;
        sd->qLaunched = NO;
        SeamSelectSlot (sd, 0);
        }
    return (YES);
}

void MB200BatchEnterChain (int chain, int phase)
{
    int d;

    for (d=0; d<numCurrentDivisions; d++)
        {
        ModelInfo *m = &modelSettings[d];
        SeamInstallScratch (m, &seamDiv[d], chain);
        if (phase == 1)
            {
            /* the division flags as this chain's move left them (ResetFlips reads them) */
            m->upDateCl   = SeamBitGet (seamFlagCl  [chain], d) ? YES : NO;
            m->upDateCijk = SeamBitGet (seamFlagCijk[chain], d) ? YES : NO;
            m->upDateAll  = SeamBitGet (seamFlagAll [chain], d) ? YES : NO;
            }
        }
}

void MB200BatchLeaveChain (int chain, int phase)
{
    int d;

    for (d=0; d<numCurrentDivisions; d++)
        {
        ModelInfo *m = &modelSettings[d];
        if (phase == 0)
            {
            SeamBitAssign (seamFlagCl  [chain], d, m->upDateCl   == YES);
            SeamBitAssign (seamFlagCijk[chain], d, m->upDateCijk == YES);
            SeamBitAssign (seamFlagAll [chain], d, m->upDateAll  == YES);
            }
        if (phase == 1 && chain < seamDiv[d].nSlots && seamDiv[d].chains[chain].nExtraFlip > 0)
            {
            /* a retry (dynamic rescaling) flipped nodes the move had not touched; ResetFlips knows nothing of them:
               the move was rejected (state[chain] is back at its pre-proposal value) -> flip them back here */
            SeamDivision *sd = &seamDiv[d];
            SeamChain    *ch = &sd->chains[chain];
            int           i;
            if (state[chain] != ch->queuedState)
                for (i=0; i<ch->nExtraFlip; i++)
                    {
                    const int node = sd->extraFlip[(size_t)chain * sd->capOps + i];
                    FlipCondLikeSpace (m, chain, node);
                    FlipNodeScalerSpace (m, chain, node);
                    }
            ch->nExtraFlip = 0;
            }
        SeamRestoreScratch (m, &seamDiv[d]);
        }
}

/* phase A: what LogLike's division loop does (src/mcmc.c:7421-7441), minus the arithmetic */
void MB200BatchQueueLogLike (int chain)
{
    int         d;
    ModelInfo  *m;

    seamRun = SEAM_RUN_QUEUED;
    for (d=0; d<numCurrentDivisions; d++)
        {
        m = &modelSettings[d];
        if (m->upDateCl != YES)
            continue;
        if (MB200LaunchLogLikeForDivision (chain, d, &(m->lnLike[2*chain + state[chain]])) == NO)
            SeamFailMove (&(m->lnLike[2*chain + state[chain]]));      /* cannot happen after MB200BatchBegin's check */
        if (abortMove == YES)
            break;
        }
    seamRun = SEAM_RUN_NOW;
}

/* one device call per division for the whole generation; the divisions overlap on the device */
void MB200BatchFlush (void)
{
    int           d;
    SeamDivision *sd;

    for (d=0; d<numCurrentDivisions; d++)
        {
        sd = &seamDiv[d];
        if (sd->nQueued == 0)
            continue;
        SeamStart (sd, sd->qEv, sd->nQueued);
        sd->qLaunched = YES;
        }
    for (d=0; d<numCurrentDivisions; d++)
        if (seamDiv[d].nQueued > 0)
            SeamFinish (&seamDiv[d]);
}

/* phase B: the chain's log likelihood, with LogLike's conventions */
MrBFlt MB200BatchFinishLogLike (int chain)
{
    int           d, q;
    ModelInfo    *m;
    SeamDivision *sd;
    MrBFlt        chainLnLike = 0.0;

    for (d=0; d<numCurrentDivisions; d++)
        {
        m  = &modelSettings[d];
        sd = &seamDiv[d];
        for (q=0; q<sd->nQueued; q++)
            if (sd->qChain[q] == chain)
                break;
        if (q < sd->nQueued && sd->qLaunched == YES)
            SeamApplyResult (d, chain, sd->qRc, sd->qLnL[q], sd->qStatus[q], &(m->lnLike[2*chain + state[chain]]));
        if (abortMove == YES)
            return MRBFLT_NEG_MAX;
        chainLnLike += m->lnLike[2*chain + state[chain]];
        }
    return chainLnLike;
}

/* ---- LaunchBEAGLELogLikeMultiPartition (src/mbbeagle.h:29, called from
 *      LaunchLogLikeForBeagleMultiPartition, src/likelihood.c:7792-7843, which has already run
 *      UpDateCijk for the divisions it passes): all of them in flight together ---------- */
void LaunchBEAGLELogLikeMultiPartition (int *divisions, int divisionCount, int chain, MrBFlt *lnL)
{
    int         i, d, hadCijk;
    ModelInfo  *m;

    (*lnL) = 0.0;
    seamRun = SEAM_RUN_DEFERRED;
    for (i=0; i<divisionCount; i++)
        {
        d = divisions[i];
        m = &modelSettings[d];
        hadCijk = m->upDateCijk;
        if (MB200SeamClosedFormModel (m) == NO)
            m->upDateCijk = NO;                 /* the caller flipped and rebuilt the cijk space already ... */
        if (hadCijk == YES && d < SEAM_MAX_DIVISIONS)
            memset (seamCijkSeen[d], 0, sizeof(seamCijkSeen[d]));   /* ... so only the upload is left */
        if (MB200LaunchLogLikeForDivision (chain, d, &(m->lnLike[2*chain + state[chain]])) == NO)
            {
            MrBayesPrint ("%s   H100 engine: division %d is outside the engine's coverage\n", spacer, d+1);
            SeamFailMove (&(m->lnLike[2*chain + state[chain]]));
            }
        m->upDateCijk = hadCijk;
        }
    seamRun = SEAM_RUN_NOW;
    SeamCollect (divisions, divisionCount, chain);
    for (i=0; i<divisionCount; i++)
        (*lnL) += modelSettings[divisions[i]].lnLike[2*chain + state[chain]];
    if (abortMove == YES)
        (*lnL) = MRBFLT_NEG_MAX;
}


/* ======================================================================================
 * Node-granular function-pointer forms (typedefs src/bayes.h:960-965; installed per division by
 * SetLikeFunctions, src/mcmc.c:17918-18327; called by the reference's own per-node loop,
 * src/likelihood.c:7892-7971).
 *
 * With these installed in ModelInfo (m->TiProbs, m->CondLikeDown, m->CondLikeRoot,
 * m->CondLikeScaler, m->Likelihood) the UNMODIFIED LaunchLogLikeForDivision drives the engine: every
 * call below records one piece of the evaluation exactly where the reference's CPU kernel would have
 * done the arithmetic -- TiProbs_* queue a P(t) rebuild, CondLikeDown_* / CondLikeRoot_* flip the
 * conditional-likelihood space like their CPU namesakes (src/likelihood.c:795) and queue a node update,
 * CondLikeScaler_* marks that node as rescaled -- and Likelihood_* closes the record and runs it as ONE
 * fused launch, returning lnL with the reference's conventions.  The driver's own FlipTiProbsSpace /
 * FlipNodeScalerSpace / FlipSiteScalerSpace calls are the index bookkeeping; its RemoveNodeScalers /
 * Copy / ResetSiteScalers calls touch only the (unused) host scaler arrays, the device does the same
 * work from scale_remove / site_scaler_src.
 * ====================================================================================== */
static void SeamOpenRecord (SeamDivision *sd, ModelInfo *m, int chain)
{
    if (sd->recording == YES && sd->recChain == chain && sd->recState == state[chain])
        return;
    sd->recording = YES;
    sd->recChain  = chain;
    sd->recState  = state[chain];
    sd->ev.matrix_update_count = 0;
    sd->ev.matrix_updates      = sd->mats;
    sd->ev.operation_count     = 0;
    sd->ev.operations          = sd->ops;
    sd->inlineEigen = MB200SeamClosedFormModel (m);
}

int TiProbs_B200 (TreeNode *p, int division, int chain)
{
    ModelInfo           *m  = &modelSettings[division];
    SeamDivision        *sd = &seamDiv[division];

    if (sd->instance < 0)
        return (ERROR);
    SeamOpenRecord (sd, m, chain);
    if (sd->stdHostP == NO && sd->ev.matrix_update_count >= sd->capMats)
        return (ERROR);
    /* the caller has flipped the branch's slot already (src/likelihood.c:7899) */
    return SeamMatrixRecord (m, sd, p, chain);
}

static int SeamRecordNode (TreeNode *p, int division, int chain, int isRoot)
{
    ModelInfo       *m  = &modelSettings[division];
    SeamDivision    *sd = &seamDiv[division];
    mb200_operation *op;

    if (sd->instance < 0)
        return (ERROR);
    SeamOpenRecord (sd, m, chain);
    if (sd->ev.operation_count >= sd->capOps)
        return (ERROR);
    op = &sd->ops[sd->ev.operation_count++];
    FlipCondLikeSpace (m, chain, p->index);
    SeamOpRecord (m, sd, op, p, chain, isRoot);
    /* the caller removes the node's old scaler right after this call when this holds
       (src/likelihood.c:7938) and flips the node-scaler space after that (:7959) */
    op->scale_remove = SeamScaleRemove (m, p, chain);
    op->scale_write  = MB200_NONE;
    return (NO_ERROR);
}

int CondLikeDown_B200 (TreeNode *p, int division, int chain)
{
    return SeamRecordNode (p, division, chain, NO);
}

int CondLikeRoot_B200 (TreeNode *p, int division, int chain)
{
    return SeamRecordNode (p, division, chain, YES);
}

int CondLikeScaler_B200 (TreeNode *p, int division, int chain)
{
    int              i;
    ModelInfo       *m  = &modelSettings[division];
    SeamDivision    *sd = &seamDiv[division];

    if (sd->instance < 0 || sd->recording == NO)
        return (ERROR);
    /* the node just recorded (the caller rescales right after computing, src/likelihood.c:7962-7965) */
    for (i=sd->ev.operation_count-1; i>=0; i--)
        if (sd->ops[i].dest == m->condLikeIndex[chain][p->index])
            break;
    if (i < 0)
        return (ERROR);
    sd->ops[i].scale_write = m->nodeScalerIndex[chain][p->index];    /* after the caller's FlipNodeScalerSpace */
    m->unscaledNodes[chain][p->index] = 0;                           /* CondLikeScaler_* (src/likelihood.c:4985) */
    return (NO_ERROR);
}

int Likelihood_B200 (TreeNode *p, int division, int chain, MrBFlt *lnL, int whichSitePats)
{
    ModelInfo       *m  = &modelSettings[division];
    SeamDivision    *sd = &seamDiv[division];

    if (sd->instance < 0)
        return (ERROR);
    SeamOpenRecord (sd, m, chain);          /* nothing dirty: root integration alone */
    sd->recording = NO;
    /* the caller has flipped the site-scaler space and reset or copied it (src/likelihood.c:7885-7889) */
    SeamSiteScalers (m, sd, chain);
    if ((sd->inlineEigen == YES) ? SeamClosedFormEigen (m, chain, sd->eigenBlock) == ERROR
                                 : (m->dataType != STANDARD && SeamSyncCijk (m, sd, division, chain) == ERROR))
        return SeamFailMove (lnL);
    SeamCategoryRates (m, sd, division, chain);
    return SeamRootAndLaunch (division, chain, p->index, lnL, whichSitePats);
}

/* What SetLikeFunctions (src/mcmc.c:17918) does for a division the engine covers: create the
 * instance and point the five hot-path function pointers at the forms above.  Call it after
 * SetLikeFunctions and InitChainCondLikes; returns ERROR (pointers untouched) for divisions
 * outside the engine's coverage. */
int MB200InstallLikeFunctions (int division)
{
    ModelInfo *m;

    SeamInit ();
    if (division < 0 || division >= numCurrentDivisions || division >= SEAM_MAX_DIVISIONS)
        return (ERROR);
    m = &modelSettings[division];
    if (MB200SeamDivisionSupported (m) == NO || InitBeagleInstance (m, division) == ERROR)
        return (ERROR);
    m->TiProbs        = &TiProbs_B200;
    m->CondLikeDown   = &CondLikeDown_B200;
    m->CondLikeRoot   = &CondLikeRoot_B200;
    m->CondLikeScaler = &CondLikeScaler_B200;
    m->Likelihood     = &Likelihood_B200;
    return (NO_ERROR);
}

/* ======================================================================================
 * Host readers of conditional-likelihood buffers (SURVEY 8f4).  CondLikeUp_* (src/likelihood.c:4574-4925),
 * PrintAncStates_* (src/mcmc.c:10713, 10902) and PrintSiteRates_Gen (src/mcmc.c:12212) work on the host arrays
 * m->condLikes / m->tiProbs / m->scalers of the cold chain at sample time (src/mcmc.c:13029, 13134-13153), through
 * function pointers.  The engine owns those buffers, so the three pointers are wrapped: the first reader call after an
 * evaluation copies the chain's CURRENT buffers (every interior node's conditional likelihoods, every branch's P(t), the
 * site scalers) from the device into the host arrays, in the reference's scalar layout [k][c][s] -- which is the
 * engine's own order -- and then the reference's reader runs unchanged.  The readers' scratch writes (the final-pass
 * vectors go to the scratch slots, src/likelihood.c:4870-4873) stay on the host.
 * ====================================================================================== */
static int SeamHostBuffersFor (ModelInfo *m, SeamDivision *sd)
{
    /* chain batching gave the chains buffer indices beyond the reference's own counts: the host tables need entries
       for them too (the reference frees its own numCondLikes / numTiProbs / numScalers entries and the table; the
       appended buffers are the seam's) */
    int     i, n = sd->extraCl + sd->extraTi + sd->extraNs;
    CLFlt **tab;

    if (n == 0 || sd->hostExtra != NULL)
        return (NO_ERROR);
    sd->hostExtra = (CLFlt **) SafeCalloc ((size_t)n, sizeof(CLFlt *));
    if (!sd->hostExtra)
        return (ERROR);
    if (sd->extraCl > 0)
        {
        tab = (CLFlt **) SafeRealloc ((void *) m->condLikes, (size_t)(m->numCondLikes + sd->extraCl) * sizeof(CLFlt *));
        if (!tab) return (ERROR);
        m->condLikes = tab;
        for (i=0; i<sd->extraCl; i++)
            if ((tab[m->numCondLikes + i] = sd->hostExtra[sd->nHostExtra++] = (CLFlt *) SafeCalloc ((size_t)m->condLikeLength, sizeof(CLFlt))) == NULL)
                return (ERROR);
        }
    if (sd->extraTi > 0)
        {
        tab = (CLFlt **) SafeRealloc ((void *) m->tiProbs, (size_t)(m->numTiProbs + sd->extraTi) * sizeof(CLFlt *));
        if (!tab) return (ERROR);
        m->tiProbs = tab;
        for (i=0; i<sd->extraTi; i++)
            if ((tab[m->numTiProbs + i] = sd->hostExtra[sd->nHostExtra++] = (CLFlt *) SafeCalloc ((size_t)m->tiProbLength, sizeof(CLFlt))) == NULL)
                return (ERROR);
        }
    if (sd->extraNs > 0)
        {
        tab = (CLFlt **) SafeRealloc ((void *) m->scalers, (size_t)(m->numScalers + sd->extraNs) * sizeof(CLFlt *));
        if (!tab) return (ERROR);
        m->scalers = tab;
        for (i=0; i<sd->extraNs; i++)
            if ((tab[m->numScalers + i] = sd->hostExtra[sd->nHostExtra++] = (CLFlt *) SafeCalloc ((size_t)m->numChars, sizeof(CLFlt))) == NULL)
                return (ERROR);
        }
    return (NO_ERROR);
}

static int SeamSyncHost (int division, int chain)
{
    ModelInfo    *m  = &modelSettings[division];
    SeamDivision *sd = &seamDiv[division];
    Tree         *t;
    TreeNode     *p;
    int           i, rc = MB200_SUCCESS;

    if (sd->instance < 0 || m->condLikes == NULL || m->tiProbs == NULL || m->scalers == NULL)
        return (ERROR);
    if (sd->syncedStamp == sd->evalStamp && sd->syncedChain == chain && sd->syncedState == state[chain])
        return (NO_ERROR);                      /* the host arrays mirror this state already */
    if (SeamHostBuffersFor (m, sd) == ERROR)
        return (ERROR);
    t = GetTree (m->brlens, chain, state[chain]);
    for (i=0; i<t->nNodes && rc == MB200_SUCCESS; i++)
        {
        p = t->allDownPass[i];
        if (p->left != NULL && p->right != NULL)
            rc = seamBackend->get_partials (sd->instance, m->condLikeIndex[chain][p->index], m->condLikes[m->condLikeIndex[chain][p->index]]);
        if (rc == MB200_SUCCESS && p->anc != NULL && m->tiProbsIndex[chain][p->index] >= 0)
            rc = seamBackend->get_transition_matrix (sd->instance, m->tiProbsIndex[chain][p->index], m->tiProbs[m->tiProbsIndex[chain][p->index]]);
        }
    if (rc == MB200_SUCCESS)
        rc = seamBackend->get_scalers (sd->instance, m->siteScalerIndex[chain], m->scalers[m->siteScalerIndex[chain]]);
    if (rc != MB200_SUCCESS)
        {
        MrBayesPrint ("%s   H100 engine: cannot read the buffers of division %d back (%s)\n", spacer, division+1, mb200_error_string (rc));
        return (ERROR);
        }
    sd->syncedStamp = sd->evalStamp; sd->syncedChain = chain; sd->syncedState = state[chain];
    return (NO_ERROR);
}

int CondLikeUp_B200 (TreeNode *p, int division, int chain)
{
    SeamDivision *sd = &seamDiv[division];
    if (sd->refCondLikeUp == NULL || SeamSyncHost (division, chain) == ERROR)
        return (ERROR);
    return sd->refCondLikeUp (p, division, chain);
}

int PrintAncStates_B200 (TreeNode *p, int division, int chain)
{
    SeamDivision *sd = &seamDiv[division];
    if (sd->refPrintAncStates == NULL || SeamSyncHost (division, chain) == ERROR)
        return (ERROR);
    return sd->refPrintAncStates (p, division, chain);
}

int PrintSiteRates_B200 (TreeNode *p, int division, int chain)
{
    SeamDivision *sd = &seamDiv[division];
    if (sd->refPrintSiteRates == NULL || SeamSyncHost (division, chain) == ERROR)
        return (ERROR);
    return sd->refPrintSiteRates (p, division, chain);
}

/* report possel=yes / siteomega=yes (codon models with omega categories): PosSelProbs and SiteOmegas (src/mcmc.c:10108, 10267)
   read the conditional likelihoods of ONE node, the root's left child, in the scalar layout [k][c][s] -- the layout
   mb200_get_partials delivers.  The SIMD builds install PosSelProbs_SSE / SiteOmegas_SSE, which expect the vector layout of
   their own kernels; the wrappers therefore call the scalar functions on the synced buffer, whatever the build. */
int PosSelProbs (TreeNode *p, int division, int chain);
int SiteOmegas (TreeNode *p, int division, int chain);

static int SeamSyncRootPartials (TreeNode *p, int division, int chain)
{
    ModelInfo    *m  = &modelSettings[division];
    SeamDivision *sd = &seamDiv[division];
    int           idx;

    if (sd->instance < 0 || m->condLikes == NULL || SeamHostBuffersFor (m, sd) == ERROR)
        return (ERROR);
    idx = m->condLikeIndex[chain][p->index];
    if (seamBackend->get_partials (sd->instance, idx, m->condLikes[idx]) != MB200_SUCCESS)
        return (ERROR);
    return (NO_ERROR);
}

int PosSelProbs_B200 (TreeNode *p, int division, int chain)
{
    if (SeamSyncRootPartials (p, division, chain) == ERROR)
        return (ERROR);
    return PosSelProbs (p, division, chain);
}

int SiteOmegas_B200 (TreeNode *p, int division, int chain)
{
    if (SeamSyncRootPartials (p, division, chain) == ERROR)
        return (ERROR);
    return SiteOmegas (p, division, chain);
}

/* what SetLikeFunctions would do for a covered division that reports ancestral states or site rates; call it after
   SetLikeFunctions (it runs for every mcmc command) -- idempotent */
int MB200InstallReaders (int division)
{
    ModelInfo    *m;
    SeamDivision *sd;

    SeamInit ();
    if (division < 0 || division >= numCurrentDivisions || division >= SEAM_MAX_DIVISIONS)
        return (ERROR);
    m  = &modelSettings[division];
    sd = &seamDiv[division];
    if (MB200SeamDivisionSupported (m) == NO)
        return (ERROR);
    if (m->printPosSel == YES || m->printSiteOmegas == YES)
        {
        m->PosSelProbs = &PosSelProbs_B200;
        m->SiteOmegas  = &SiteOmegas_B200;
        sd->omegaReaders = YES;
        }
    if (SeamReadersWanted (m) == NO)
        return (sd->omegaReaders == YES) ? NO_ERROR : ERROR;
    if (m->CondLikeUp != &CondLikeUp_B200 && m->CondLikeUp != NULL)
        { sd->refCondLikeUp = m->CondLikeUp; m->CondLikeUp = &CondLikeUp_B200; }
    if (m->PrintAncStates != &PrintAncStates_B200 && m->PrintAncStates != NULL)
        { sd->refPrintAncStates = m->PrintAncStates; m->PrintAncStates = &PrintAncStates_B200; }
    if (m->PrintSiteRates != &PrintSiteRates_B200 && m->PrintSiteRates != NULL)
        { sd->refPrintSiteRates = m->PrintSiteRates; m->PrintSiteRates = &PrintSiteRates_B200; }
    sd->readers = YES;
    sd->syncedStamp = -1;
    return (NO_ERROR);
}

/* ---- InitBeagleMultiPartitionInstance (src/mbbeagle.h:28, src/mbbeagle.c:1500): one instance per
 *      division; unlike BEAGLE's single multi-partition instance the divisions need not share their
 *      dimensions (src/mbbeagle.c:1522-1546), and they may live on different GPUs ------------- */
int InitBeagleMultiPartitionInstance (void)
{
    int d, nOk = 0;

    for (d=0; d<numCurrentDivisions; d++)
        if (MB200SeamDivisionSupported (&modelSettings[d]) == YES)
            {
            if (InitBeagleInstance (&modelSettings[d], d) == ERROR)
                return (ERROR);
            nOk++;
            }
    return (nOk > 0) ? NO_ERROR : ERROR;
}

/* ---- recalculateScalers (src/mbbeagle.h:16, src/mbbeagle.c:541): rebuild every scaler of a chain's
 *      current state.  The engine rescales every node (the built-in path's policy), so this is one
 *      full evaluation of each division with the site scalers reset: all interior nodes recomputed
 *      into their scratch slots and flipped in, like TreeCondLikes_Beagle_Rescale_All. ------------ */
void recalculateScalers (int chain)
{
    int         d, i;
    ModelInfo  *m;
    Tree       *tree;
    TreeNode   *p;
    MrBFlt      lnL;
    int         savedAll, savedCl, savedAbort = abortMove;

    for (d=0; d<numCurrentDivisions; d++)
        {
        m = &modelSettings[d];
        if (MB200SeamDivisionSupported (m) == NO || d >= SEAM_MAX_DIVISIONS || seamDiv[d].instance < 0)
            continue;
        tree = GetTree (m->brlens, chain, state[chain]);
        savedAll = m->upDateAll;
        savedCl  = m->upDateCl;
        for (i=0; i<tree->nIntNodes; i++)
            {
            p = tree->intDownPass[i];
            p->upDateCl = YES;
            }
        m->upDateAll = YES;                 /* ResetSiteScalers instead of CopySiteScalers */
        MB200LaunchLogLikeForDivision (chain, d, &lnL);
        m->upDateAll = savedAll;
        m->upDateCl  = savedCl;
        }
    abortMove = savedAbort;
}
