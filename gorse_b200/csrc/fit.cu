// fit.cu -- host-side mirror of cf.BPR.Fit / cf.ALS.Fit (model/cf/model.go:408-530, 609-775) above the
// per-epoch entry points: Init, Evaluate at epoch 0, epoch loop, Evaluate every `verbose` epochs and on the last
// one, early stopping on `patience`, progress / cancellation callback (monitor span.Add(1) and ctx.Err()).
// The Go shim can call this once per Fit, or drive the per-epoch entry points itself and keep the loop in Go.
// gorse_b200_cf_fit_trials runs the same loop for the trials of a model search at once.
#include <algorithm>
#include <vector>

#include "cf.cuh"
#include "tables.cuh"

using namespace gb;

namespace {

struct EvalSets {
    const int64_t *test_off;
    const int32_t *test_items;
    const int64_t *neg_off;
    const int32_t *neg_items;
};

// One fit's bookkeeping, shared by the solo fit and the model search: the (epoch, NDCG) list (model.go:434,499), the cross
// validation cadence (:496 / :741), early stopping on `patience` with the first-maximum rule (:508-517), and the result.
struct FitState {
    const gorse_b200_fit_params *p;
    std::vector<std::pair<int32_t, float>> scores;
    float score[3] = {0.f, 0.f, 0.f};   // the last evaluation
    int32_t epochs_run = 0, best_epoch = 0;
    bool early_stopped = false, cancelled = false;

    explicit FitState(const gorse_b200_fit_params *params) : p(params) {}
    // epoch `epoch` has run; whether it is evaluated
    bool ran(int32_t epoch)
    {
        epochs_run = epoch;
        return (p->verbose > 0 && epoch % p->verbose == 0) || epoch == p->n_epochs;
    }
    void record(int32_t epoch, const float s[3])
    {
        score[0] = s[0]; score[1] = s[1]; score[2] = s[2];
        scores.emplace_back(epoch, s[0]);
    }
    // after an evaluated epoch: no improvement in the last `patience` epochs stops the fit
    bool stops(int32_t epoch)
    {
        if (p->patience <= 0 || epoch <= p->patience) return false;
        // lo.MaxBy with a.B > b.B keeps the FIRST maximum
        std::pair<int32_t, float> best = scores[0];
        for (auto &s : scores) if (s.second > best.second) best = s;
        if (best.first > epoch - p->patience) return false;
        early_stopped = true;
        best_epoch = best.first;
        return true;
    }
    // span.Add(1) + ctx cancellation (model.go:490-493,519): a cancelled fit returns Score{}
    void cancel() { cancelled = true; }
    gorse_b200_fit_result result() const
    {
        gorse_b200_fit_result r{};
        r.epochs_run = epochs_run;
        if (cancelled) { r.cancelled = 1; return r; }
        r.ndcg = score[0]; r.precision = score[1]; r.recall = score[2];
        r.early_stopped = early_stopped;
        r.best_epoch = best_epoch;
        return r;
    }
};

// Evaluate's inputs go to the device once per Fit; without caller-sampled negatives they are drawn there
// (testSet.SampleUserNegatives(trainSet, Candidates) with NewRandomGenerator(0), evaluator.go:42, dataset.go:244)
struct Plan {
    gorse_b200_eval *p = nullptr;
    ~Plan() { gorse_b200_eval_destroy(p); }
    int32_t create(gorse_b200_cf *cf, const EvalSets &ev, const gorse_b200_fit_params *fp)
    {
        return gorse_b200_eval_create(cf, ev.test_off, ev.test_items, ev.neg_off, ev.neg_items, fp->candidates, 0, fp->topk, &p);
    }
};

int32_t fit_loop(gorse_b200_cf *cf, bool als, const gorse_b200_fit_params *p, const EvalSets &ev, gorse_b200_progress_fn progress,
                 void *user, gorse_b200_fit_result *res)
{
    float score[3] = {0.f, 0.f, 0.f};
    FitState st(p);
    *res = gorse_b200_fit_result{};
    // Init (model.go:414 / :615)
    GB_TRY(gorse_b200_cf_init_normal(cf, p->init_mean, p->init_stddev, p->seed));
    Plan plan;
    GB_TRY(plan.create(cf, ev, p));
    GB_TRY(gorse_b200_eval_run(plan.p, score));  // :433 / :630
    st.record(0, score);
    for (int32_t epoch = 1; epoch <= p->n_epochs; epoch++) {
        if (als) GB_TRY(gorse_b200_als_epoch(cf, p->reg, p->alpha));
        else GB_TRY(gorse_b200_bpr_epoch(cf, p->lr, p->reg, cf->n_feedback_global, p->seed + (uint64_t)epoch, GORSE_B200_SCATTER_ATOMIC));
        const bool evaluated = st.ran(epoch);
        if (evaluated) {
            GB_TRY(gorse_b200_eval_run(plan.p, score));
            st.record(epoch, score);
        }
        if (progress && progress(user, epoch, p->n_epochs, evaluated ? score[0] : -1.0f) != 0) {
            st.cancel();
            break;
        }
        if (evaluated && st.stops(epoch)) break;
    }
    GB_TRY(gorse_b200_ctx_sync(cf->ctx));
    *res = st.result();
    return GORSE_B200_OK;
}

// ModelSearch's trials in one loop: every epoch runs the live BPR trials in one bpr_trials_epoch and each live ALS trial's
// epoch, then evaluates and checks each trial exactly as fit_loop does
int32_t fit_trials(gorse_b200_cf *cf, int32_t n, const int32_t *als, const gorse_b200_fit_params *tp, const EvalSets &ev,
                   gorse_b200_trials_progress_fn progress, void *user, gorse_b200_fit_result *results, float *const *P_out,
                   float *const *Q_out)
{
    gorse_b200_ctx *c = cf->ctx;
    Plan plan;
    GB_TRY(plan.create(cf, ev, &tp[0]));   // checks the test and negative rows before the device is touched
    std::vector<DevBuf<float>> tP((size_t)n), tQ((size_t)n);   // each trial's factor tables
    std::vector<FitState> st;
    std::vector<bool> done((size_t)n, false);
    float score[3];
    for (int32_t k = 0; k < n; k++) {
        st.emplace_back(&tp[k]);
        GB_TRY(tP[k].alloc(cf->P.n));
        GB_TRY(tQ[k].alloc(cf->Q.n));
        GB_TRY(init_normal_tables(cf, tP[k].p, tQ[k].p, tp[k].init_mean, tp[k].init_stddev, tp[k].seed));
        GB_TRY(eval_run_tables(plan.p, tP[k].p, tQ[k].p, score));
        st[k].record(0, score);
        done[k] = tp[k].n_epochs == 0;
    }
    std::vector<gorse_b200_trial_state> states((size_t)n);
    std::vector<float *> bP, bQ;
    std::vector<float> blr, breg;
    for (int32_t epoch = 1; std::find(done.begin(), done.end(), false) != done.end(); epoch++) {
        bP.clear(); bQ.clear(); blr.clear(); breg.clear();
        for (int32_t k = 0; k < n; k++)
            if (!done[k] && !als[k]) { bP.push_back(tP[k].p); bQ.push_back(tQ[k].p); blr.push_back(tp[k].lr); breg.push_back(tp[k].reg); }
        GB_TRY(bpr_trials_epoch(cf, (int)bP.size(), bP.data(), bQ.data(), blr.data(), breg.data(), tp[0].seed + (uint64_t)epoch));
        for (int32_t k = 0; k < n; k++)
            if (!done[k] && als[k]) GB_TRY(als_epoch_tables(cf, tP[k].p, tQ[k].p, tp[k].reg, tp[k].alpha));
        for (int32_t k = 0; k < n; k++) {
            gorse_b200_trial_state &s = states[k];
            s.ndcg = -1.0f;
            if (!done[k]) {
                const bool evaluated = st[k].ran(epoch);
                if (evaluated) {
                    GB_TRY(eval_run_tables(plan.p, tP[k].p, tQ[k].p, score));
                    st[k].record(epoch, score);
                    s.ndcg = score[0];
                }
                done[k] = (evaluated && st[k].stops(epoch)) || epoch == tp[k].n_epochs;
            }
            s.epochs_run = st[k].epochs_run;
            s.finished = done[k];
        }
        if (progress && progress(user, epoch, n, states.data()) != 0) {
            for (int32_t k = 0; k < n; k++)
                if (!done[k]) { st[k].cancel(); done[k] = true; }
        }
    }
    GB_TRY(gorse_b200_ctx_sync(c));
    for (int32_t k = 0; k < n; k++) {
        results[k] = st[k].result();
        if (P_out && P_out[k] && cf->P.n)
            GB_CUDA(cudaMemcpyAsync(P_out[k], tP[k].p, cf->P.n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
        if (Q_out && Q_out[k] && cf->Q.n)
            GB_CUDA(cudaMemcpyAsync(Q_out[k], tQ[k].p, cf->Q.n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    }
    GB_CUDA(cudaStreamSynchronize(c->stream));
    return GORSE_B200_OK;
}

int32_t check_params(const gorse_b200_fit_params *p, const gorse_b200_fit_result *res)
{
    GB_CHECK_ARG(p != nullptr && res != nullptr, "NULL params/result");
    GB_CHECK_ARG(p->n_epochs >= 0, "negative n_epochs");
    GB_CHECK_ARG(p->topk >= 1, "topk must be >= 1");
    GB_CHECK_ARG(p->candidates >= 0, "negative candidates");
    return GORSE_B200_OK;
}

}  // namespace

extern "C" {

int32_t gorse_b200_fit_params_default(int32_t als, gorse_b200_fit_params *p)
{
    GB_CHECK_ARG(p != nullptr, "params is NULL");
    *p = gorse_b200_fit_params{};
    // BPR.SetParams model.go:389-394 / ALS.SetParams :580-585; FitConfig NewFitConfig :58-65
    p->n_factors = 16;
    p->n_epochs = als ? 50 : 100;
    p->lr = 0.05f;
    p->reg = als ? 0.06f : 0.01f;
    p->init_mean = 0.f;
    p->init_stddev = als ? 0.1f : 0.001f;
    p->alpha = 0.001f;
    p->seed = 0;
    p->verbose = 10;
    p->candidates = 100;
    p->topk = 10;
    p->patience = 0;
    return GORSE_B200_OK;
}

int32_t gorse_b200_bpr_fit(gorse_b200_cf *cf, const gorse_b200_fit_params *params, const int64_t *test_off,
                           const int32_t *test_items, const int64_t *neg_off, const int32_t *neg_items,
                           gorse_b200_progress_fn progress, void *user, gorse_b200_fit_result *result)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    GB_TRY(check_params(params, result));
    EvalSets ev{test_off, test_items, neg_off, neg_items};
    return fit_loop(cf, false, params, ev, progress, user, result);
}

int32_t gorse_b200_als_fit(gorse_b200_cf *cf, const gorse_b200_fit_params *params, const int64_t *test_off,
                           const int32_t *test_items, const int64_t *neg_off, const int32_t *neg_items,
                           gorse_b200_progress_fn progress, void *user, gorse_b200_fit_result *result)
{
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    GB_TRY(check_params(params, result));
    EvalSets ev{test_off, test_items, neg_off, neg_items};
    return fit_loop(cf, true, params, ev, progress, user, result);
}

int32_t gorse_b200_cf_fit_trials(gorse_b200_cf *cf, int32_t n_trials, const int32_t *als, const gorse_b200_fit_params *trials,
                                 const int64_t *test_off, const int32_t *test_items, const int64_t *neg_off,
                                 const int32_t *neg_items, gorse_b200_trials_progress_fn progress, void *user,
                                 gorse_b200_fit_result *results, float *const *P_out, float *const *Q_out)
{
    // ModelSearch.Objective (model/cf/optimize.go:61-81) per trial, for the study of optimizeCollaborativeFiltering
    // (master/tasks.go:1268-1316): one FitConfig and one RandomState for every trial
    GB_CHECK_ARG(n_trials >= 1, "n_trials must be >= 1, not %d", n_trials);
    GB_CHECK_ARG(als != nullptr && trials != nullptr && results != nullptr, "NULL als/trials/results");
    for (int32_t k = 0; k < n_trials; k++) GB_TRY(check_params(&trials[k], &results[k]));
    const gorse_b200_fit_params &a = trials[0];
    for (int32_t k = 1; k < n_trials; k++) {
        const gorse_b200_fit_params &t = trials[k];
        GB_CHECK_ARG(t.n_factors == a.n_factors && t.seed == a.seed && t.verbose == a.verbose && t.candidates == a.candidates &&
                         t.topk == a.topk && t.patience == a.patience,
                     "trial %d: n_factors, seed, verbose, candidates, topk and patience must equal trial 0's", k);
    }
    GB_CHECK_ARG(cf != nullptr, "cf is NULL");
    GB_CHECK_ARG(a.n_factors == cf->d, "n_factors %d is not the model's d = %d", a.n_factors, cf->d);
    if (cf->ctx->world > 1) { set_error("fit_trials runs on one GPU"); return GORSE_B200_ERR_UNSUPPORTED; }
    for (int32_t k = 0; k < n_trials; k++) {
        if (als[k] && !cf->has_item_csr) { set_error("trial %d: ALS needs the item CSR (item_off/item_users) at cf_create", k); return GORSE_B200_ERR_STATE; }
        if (!als[k] && cf->d != 16 && cf->d != 32 && cf->d != 64 && cf->d != 128) {
            set_error("trial %d: batched BPR trials need d in {16, 32, 64, 128}, not %d", k, cf->d);
            return GORSE_B200_ERR_UNSUPPORTED;
        }
    }
    ScopedDevice sd(cf->ctx->device);
    EvalSets ev{test_off, test_items, neg_off, neg_items};
    return fit_trials(cf, n_trials, als, trials, ev, progress, user, results, P_out, Q_out);
}

}  // extern "C"
