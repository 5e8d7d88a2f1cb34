/*
 * pruning_oracle.h -- TEST INFRASTRUCTURE: CPU restatement of MrBayes' tree-likelihood
 * hot path, used ONLY as the checker in tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline leg.  The product (libmb200.so) never links, loads or calls this.
 *
 * Pinned against the reference itself: tests/golden/ holds evaluation records produced by
 * the unmodified reference (oracle/ref_harness.c); tests/test_oracle_golden.py replays
 * them through this file and demands the reference's lnL to <= 1e-12 relative.
 *
 * The API mirrors include/mb200.h one to one (same structs, orc_ prefix) so a test can feed
 * identical inputs to the oracle and to the CUDA engine.
 */
#ifndef PRUNING_ORACLE_H_
#define PRUNING_ORACLE_H_

#include "mb200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* float arithmetic family to restate (they differ in rounding only) */
#define ORC_ARITH_MULADD 0   /* scalar / SSE / AVX variants: separate multiply and add     */
#define ORC_ARITH_FMA    1   /* CondLikeDown_NUC4_FMA etc.: fused multiply-add, logf scaler */

int orc_create_instance   (const mb200_instance_config *config, int *instance);
int orc_finalize_instance (int instance);
int orc_set_arith         (int instance, int arith);
int orc_set_tip_states      (int instance, int tip, const uint64_t *state_masks);
int orc_set_pattern_weights (int instance, int row, const float *weights);
int orc_set_pattern_states  (int instance, const int *state_counts, const int *matrix_offsets,
                             const int *freq_offsets, int matrix_length, int dummy_patterns,
                             int uncompressed_sites);
int orc_set_cijk (int instance, int eigen, const double *block);
int orc_set_eigen_decomposition (int instance, int eigen, const double *eigvecs,
                                 const double *inverse_eigvecs, const double *eigvals);
int orc_evaluate (int instance, const mb200_evaluation *evaluations, int count,
                  double *lnL, int *status);
int orc_get_partials          (int instance, int buffer, float *out);
int orc_set_partials          (int instance, int buffer, const float *in);
int orc_get_transition_matrix (int instance, int matrix, float *out);
int orc_set_transition_matrix (int instance, int matrix, const float *in);
int orc_get_scalers           (int instance, int scaler, float *out);
int orc_set_scalers           (int instance, int scaler, const float *in);
long long orc_cl_updates      (int instance);   /* node*pattern*rate updates done so far */

/* Site-pattern compression (CompressData, src/model.c:2466-2782), integer, bit-exact:
 * columns of an nTaxa x nSites matrix of state-set codes are merged into the first earlier
 * identical column; returns the number of unique patterns, pattern_of_site[nSites],
 * first_site_of_pattern[<=nSites] and weights[<=nSites] (site counts). */
int orc_compress_patterns (const uint64_t *matrix, int n_taxa, int n_sites,
                           int *pattern_of_site, int *first_site_of_pattern, int *weights);

#ifdef __cplusplus
}
#endif
#endif
