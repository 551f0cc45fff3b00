// recall.cu -- batched collaborative-filtering recall: gorse_b200_vecdb_query_excluding.
//
// The worker's CF recall (worker/pipeline.go:403-449) asks, per user, QueryVectors(user embedding, topK = n + |E_u|) and then
// drops the user's feedback items E_u (logics/recommend.go:67-80).  Here one call answers many users: row q's answer is the
// first k_q = n + |E_q| allowed slots by (score desc, slot asc), minus the slots in E_q, with the scores of
// gorse_b200_vecdb_query, bit for bit.  This file checks the arguments and prepares the exclusion lists; the rows run through
// the index's top-k pipeline (recall::recall_rows, topk.cu).
#include "stages.cuh"

using namespace gb;

extern "C" int32_t gorse_b200_vecdb_query_excluding(gorse_b200_vecdb *db, int64_t nq, const float *q_values, const int32_t *categories,
                                                    int32_t n_categories, int32_t n, const int64_t *excl_off, const int64_t *excl_slots,
                                                    int64_t *slots_out, float *scores_out, int32_t *count_out, int64_t *exact_rows_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    GB_CHECK_ARG(nq >= 0 && n_categories >= 0, "negative count");
    if (exact_rows_out) *exact_rows_out = 0;
    if (nq == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(count_out != nullptr && excl_off != nullptr, "count_out / excl_off is NULL");
    GB_CHECK_ARG(excl_off[0] == 0, "excl_off[0] must be 0");
    for (int64_t q = 0; q < nq; q++)
        GB_CHECK_ARG(excl_off[q + 1] >= excl_off[q], "excl_off not non-decreasing at %lld", (long long)q);
    GB_CHECK_ARG(excl_off[nq] == 0 || excl_slots != nullptr, "excl_slots is NULL");
    if (db->dim == 0) {
        set_error("query_excluding serves dense collections only");
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    if (n <= 0) {
        for (int64_t q = 0; q < nq; q++) count_out[q] = 0;
        return GORSE_B200_OK;
    }
    GB_CHECK_ARG(q_values != nullptr && slots_out != nullptr && scores_out != nullptr, "NULL query / output");
    GB_CHECK_ARG(n_categories == 0 || categories != nullptr, "categories is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    const int64_t n_slots = (int64_t)db->ts.size();
    for (int64_t q = 0; q < nq; q++)
        GB_CHECK_ARG((int64_t)n + (excl_off[q + 1] - excl_off[q]) <= INT32_MAX, "row %lld: n + |E| overflows", (long long)q);
    // each row's exclusions once, sorted, -1 entries dropped (they still count in k_q)
    std::vector<int64_t> ex, ex_off;
    GB_TRY(exclusion_rows(nq, excl_off, excl_slots, n_slots, "row", "slot", ex, ex_off));
    if (n_slots == 0) {
        for (int64_t q = 0; q < nq; q++) count_out[q] = 0;
        return GORSE_B200_OK;
    }
    ScopedDevice sd(db->ctx->device);
    GB_TRY(vecdb_allow(db, categories, n_categories));
    std::lock_guard<std::mutex> lk2(db->dense->mu);
    return recall::recall_rows(db->dense, db->d_allow.p, nq, q_values, nullptr, n, excl_off, ex.data(), ex_off.data(), nullptr, slots_out, scores_out, count_out,
                               exact_rows_out);
}
