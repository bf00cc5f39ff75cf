/* crb_oracle_slp.h — CPU restatement of the samplers and the lookup-table search of src/state_lattice_planner.cpp.
 * TEST INFRASTRUCTURE ONLY. */
#ifndef CRB_ORACLE_SLP_H_
#define CRB_ORACLE_SLP_H_
#include <stdint.h>

#include "../include/crb.h" /* crb_slp_sampler, the CRB_SLP_* kinds, limits and statuses: the same rules as the kernel */
#ifdef __cplusplus
extern "C" {
#endif

/* The samplers with the layout and outputs of crb_slp_sample_states_batched (host pointers; status may be NULL).
 * The sampler must be valid (crb_slp_states_per_query >= 0); S is its states per query.  nthreads <= 0 means all
 * cores. */
void crb_oracle_slp_sample(int64_t n_q, const crb_slp_sampler* s, int S, const float* qp, float* target,
                           int32_t* n_states, int32_t* status, int nthreads);
/* search_nearest_one_from_lookuptable with the layout and outputs of crb_slp_search_nearest_batched (k0 and row may
 * be NULL) */
void crb_oracle_slp_search(int64_t n, const float* target, const float* table, int rows, const float* k0,
                           float* param, int32_t* row, int nthreads);

#ifdef __cplusplus
}
#endif
#endif
