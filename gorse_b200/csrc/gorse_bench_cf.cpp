// gorse-bench cf -- the collaborative-filtering sub-command the reference's cmd/gorse-bench is missing (SURVEY 8f-3, F2):
// load an NCF-format dataset like dataset.LoadDataFromBuiltIn (dataset/dataset.go:398-490), fit BPR or ALS like
// master.newCollaborativeFilteringModel would (model/cf/model.go:408-530, 609-775) and print the tables cmd/gorse-bench
// prints for its other sub-commands (cmd/gorse-bench/main.go:517-555: dataset sizes, then NDCG / Precision / Recall).
// Plain C++ over the C ABI of libgorse_b200.so -- the calls a Go `benchCFCmd` would make through cgo.  No CPU fallback:
// without an H100 the fit fails loudly.
//
//   gorse-bench-cf --train ml-100k.train.rating --test ml-100k.test.negative [--model bpr|als] [--factors 16] [--epochs 100]
//                  [--lr 0.05] [--reg 0.01] [--alpha 0.001] [--top 10] [--verbose 10] [--seed 0] [--device 0]
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "gorse_b200.h"

static void die(const char *what)
{
    fprintf(stderr, "gorse-bench cf: %s: %s\n", what, gorse_b200_last_error());
    exit(1);
}
#define CHECK(call, what) do { if ((call) != GORSE_B200_OK) die(what); } while (0)

static int32_t progress(void *user, int32_t epoch, int32_t n_epochs, float ndcg)
{
    if (ndcg >= 0) fprintf(stderr, "epoch %d/%d  NDCG@k %.4f\n", epoch, n_epochs, ndcg);   // the reference logs at Verbose cadence
    return 0;
}

int main(int argc, char **argv)
{
    std::string train, test, model = "bpr";
    int device = 0, top = 10;
    bool have[8] = {false};
    double lr = 0, reg = 0, alpha = 0;
    int factors = 0, epochs = 0, verbose = 0;
    unsigned long long seed = 0;
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        auto val = [&]() -> const char * { if (i + 1 >= argc) { fprintf(stderr, "missing value for %s\n", a.c_str()); exit(2); } return argv[++i]; };
        if (a == "--train") train = val();
        else if (a == "--test") test = val();
        else if (a == "--model") model = val();
        else if (a == "--factors") { factors = atoi(val()); have[0] = true; }
        else if (a == "--epochs") { epochs = atoi(val()); have[1] = true; }
        else if (a == "--lr") { lr = atof(val()); have[2] = true; }
        else if (a == "--reg") { reg = atof(val()); have[3] = true; }
        else if (a == "--alpha") { alpha = atof(val()); have[4] = true; }
        else if (a == "--verbose") { verbose = atoi(val()); have[5] = true; }
        else if (a == "--top" || a == "-k") top = atoi(val());
        else if (a == "--seed") seed = strtoull(val(), nullptr, 10);
        else if (a == "--device") device = atoi(val());
        else { fprintf(stderr, "usage: gorse-bench-cf --train FILE --test FILE [--model bpr|als] [--factors N] [--epochs N] [--lr X] [--reg X] [--alpha X] [--top K] [--verbose N] [--seed S] [--device D]\n"); return 2; }
    }
    if (train.empty() || (model != "bpr" && model != "als")) { fprintf(stderr, "gorse-bench cf: --train is required, --model is bpr or als\n"); return 2; }
    const bool als = model == "als";

    gorse_b200_ncf *ds = nullptr;
    CHECK(gorse_b200_ncf_load(train.c_str(), test.empty() ? nullptr : test.c_str(), &ds), "load dataset");
    int32_t U = 0, I = 0;
    int64_t n_train = 0, n_test = 0, n_neg = 0;
    CHECK(gorse_b200_ncf_shape(ds, &U, &I, &n_train, &n_test, &n_neg), "shape");
    std::vector<int64_t> tr_off(U + 1), te_off(U + 1), ng_off(U + 1);
    std::vector<int32_t> tr_items(n_train), te_items(n_test), ng_items(n_neg);
    CHECK(gorse_b200_ncf_get(ds, tr_off.data(), tr_items.data(), te_off.data(), te_items.data(), ng_off.data(), ng_items.data()), "get");
    gorse_b200_ncf_free(ds);
    printf("+-------+--------+--------+---------------+\n|       | #users | #items | #interactions |\n+-------+--------+--------+---------------+\n");
    printf("| train | %6d | %6d | %13lld |\n| test  | %6d | %6d | %13lld |\n+-------+--------+--------+---------------+\n", U, I, (long long)n_train, U, I,
           (long long)n_test);

    // the item CSR ALS needs (dataset.GetItemFeedback: users in append order)
    std::vector<int64_t> it_off(I + 1, 0);
    std::vector<int32_t> it_users(n_train);
    if (als) {
        for (int64_t t = 0; t < n_train; t++) it_off[tr_items[t] + 1]++;
        for (int32_t i = 0; i < I; i++) it_off[i + 1] += it_off[i];
        std::vector<int64_t> cur(it_off.begin(), it_off.end() - 1);
        for (int32_t u = 0; u < U; u++)
            for (int64_t t = tr_off[u]; t < tr_off[u + 1]; t++) it_users[cur[tr_items[t]]++] = u;
    }

    gorse_b200_fit_params p;
    CHECK(gorse_b200_fit_params_default(als ? 1 : 0, &p), "params");
    if (have[0]) p.n_factors = factors;
    if (have[1]) p.n_epochs = epochs;
    if (have[2]) p.lr = (float)lr;
    if (have[3]) p.reg = (float)reg;
    if (have[4]) p.alpha = (float)alpha;
    if (have[5]) p.verbose = verbose;
    p.topk = top;
    p.seed = seed;

    gorse_b200_ctx *ctx = nullptr;
    CHECK(gorse_b200_ctx_create(device, &ctx), "context (this tool needs an H100: there is no CPU fallback)");
    gorse_b200_cf *cf = nullptr;
    auto t0 = std::chrono::steady_clock::now();
    CHECK(gorse_b200_cf_create(ctx, U, I, p.n_factors, tr_off.data(), tr_items.data(), als ? it_off.data() : nullptr, als ? it_users.data() : nullptr, &cf),
          "cf_create");
    gorse_b200_fit_result res;
    // the test file's own negatives when it has them (the NCF protocol: 99 per user), else sampled on the device
    const bool own_neg = n_neg > 0;
    if (als) CHECK(gorse_b200_als_fit(cf, &p, te_off.data(), te_items.data(), own_neg ? ng_off.data() : nullptr, own_neg ? ng_items.data() : nullptr, progress, nullptr, &res), "als_fit");
    else CHECK(gorse_b200_bpr_fit(cf, &p, te_off.data(), te_items.data(), own_neg ? ng_off.data() : nullptr, own_neg ? ng_items.data() : nullptr, progress, nullptr, &res), "bpr_fit");
    std::vector<float> P((size_t)U * p.n_factors), Q((size_t)I * p.n_factors);
    CHECK(gorse_b200_cf_get_factors(cf, P.data(), Q.data()), "get_factors");
    const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    int64_t launches = 0;
    gorse_b200_ctx_launch_count(ctx, &launches);
    printf("+-------+---------+--------------+-----------+----------+--------+\n| Model | NDCG@%-2d | Precision@%-2d | Recall@%-2d | epochs   | sec    |\n", top, top, top);
    printf("+-------+---------+--------------+-----------+----------+--------+\n| %-5s | %7.4f | %12.4f | %9.4f | %8d | %6.2f |\n", als ? "ALS" : "BPR", res.ndcg,
           res.precision, res.recall, res.epochs_run, sec);
    printf("+-------+---------+--------------+-----------+----------+--------+\n");
    const double steps = als ? 2.0 * (double)n_train * res.epochs_run : (double)n_train * res.epochs_run;
    printf("%s: %.3g %s/s end to end (create + fit + factor download), %lld kernel launches\n", als ? "eALS" : "BPR", steps / sec,
           als ? "feedback visits" : "triples", (long long)launches);
    gorse_b200_cf_destroy(cf);
    gorse_b200_ctx_destroy(ctx);
    return 0;
}
