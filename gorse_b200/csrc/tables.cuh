// tables.cuh -- the CF epoch, init and evaluation on factor tables other than the model's own P and Q.
// The public entries call these with cf->P / cf->Q; gorse_b200_cf_fit_trials (fit.cu) with the tables of each trial.
// P has the shard's user rows and Q all item rows, both d floats per row, like cf->P and cf->Q.
#pragma once
#include "cf.cuh"

namespace gb {

// cf.cu: gorse_b200_cf_init_normal's draws into P and Q
int32_t init_normal_tables(gorse_b200_cf *cf, float *P, float *Q, float mean, float stddev, uint64_t seed);
// als.cu: one eALS epoch (gorse_b200_als_epoch) on P and Q; synchronises the stream
int32_t als_epoch_tables(gorse_b200_cf *cf, float *P, float *Q, float reg, float alpha);
// evaluate.cu: gorse_b200_eval_run scoring P and Q
int32_t eval_run_tables(gorse_b200_eval *ev, const float *P, const float *Q, float *out);
// bpr.cu: one atomic round epoch of cf->n_feedback_global steps at `seed` for each of the n models (P[m], Q[m], lr[m],
// reg[m]), sampling every triple once for all of them; d in {16, 32, 64, 128}, one rank
int32_t bpr_trials_epoch(gorse_b200_cf *cf, int n, float *const *P, float *const *Q, const float *lr, const float *reg, uint64_t seed);

}  // namespace gb
