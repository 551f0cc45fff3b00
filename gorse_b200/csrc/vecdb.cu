// vecdb.cu -- one vector COLLECTION of a vectors.Database on the GPU (SURVEY 8f-1): what item-to-item, user-to-user and
// CF retrieval query in this snapshot (storage/vectors/database.go:107-120; backend semantics restated from the reference's
// default backend storage/vectors/xvec.go:288-449).
//
//   AddVectors (:288-318, an upsert by id)   gorse_b200_vecdb_add      append; the previous version of an id is tombstoned
//   GetVectors (:320-363)                    gorse_b200_vecdb_get
//   DeleteVectors(timestamp) (:365-371)      gorse_b200_vecdb_delete_before   tombstone ts < timestamp
//   CountVectors (:274-286)                  gorse_b200_vecdb_count
//   QueryVectors(q, categories, topK) (:373-449)  gorse_b200_vecdb_query
//       filter  hidden = false AND categories CONTAIN_ALL (...)  (:381-389)  -> a per-vector allow mask built on the device
//       dense   brute force over the stored fp32 vectors (exact: the reference's DiskANN is approximate), in the
//               summation order of floats.Dot / floats.Euclidean; sparse (dimension 0, Dot only, :244-248) through sparse.cu
//       score   "higher = more similar" (database.go:101): Dot -> the dot product; Euclidean / Cosine -> the NEGATED distance
//               (:425-427); sparse results with score 0 are dropped (:421-423)
// Ids are strings in the reference; the shim keeps the id <-> slot map (go/storage/vectors/b200.go) and the category
// string <-> int32 map, the library works on slots (int64, in insertion order) and category ids.
#include <algorithm>

#include <cub/cub.cuh>

#include "cf.cuh"
#include "sparse.cuh"
#include "vecdb.cuh"

extern "C" {
int32_t gorse_b200_sparse_index_create(gorse_b200_ctx *ctx, gorse_b200_sparse_index **out);
int32_t gorse_b200_sparse_index_destroy(gorse_b200_sparse_index *ix);
}

namespace gb {

// allow[i] = !blocked[i] && categories(i) contains every wanted category
__global__ void vecdb_allow_kernel(const uint8_t *blocked, const int64_t *cat_off, const int32_t *cats, const int32_t *want, int n_want,
                                   int64_t n, uint8_t *allow)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool ok = blocked[i] == 0;
    for (int w = 0; w < n_want && ok; w++) {
        bool has = false;
        for (int64_t t = cat_off[i]; t < cat_off[i + 1] && !has; t++) has = cats[t] == want[w];
        ok = has;
    }
    allow[i] = ok ? 1 : 0;
}

// flag[item] = 1 for every item with >= 1 training feedback (IsItemPredictable, model/cf/model.go:129-146)
__global__ void vecdb_mark_items_kernel(const int32_t *user_items, int64_t n, int32_t *flag)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += st) flag[user_items[i]] = 1;
}
// flag[s] = 1 for a live slot, flag[n] = 0: the input of the exclusive scan that renumbers the slots
__global__ void vecdb_live_kernel(const uint8_t *dead, int64_t n, int64_t *flag)
{
    const int64_t st = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += st) flag[i] = i < n && dead[i] == 0;
}

// device bytes held by the collection, its index, its work buffers and its neighbour cache
static int64_t vecdb_bytes(const gorse_b200_vecdb *db)
{
    return (int64_t)(db->d_blocked.bytes() + db->d_allow.bytes() + db->d_cat_off.bytes() + db->d_cats.bytes() + db->d_want.bytes() +
                     db->stage.bytes() + db->ncache.bytes() + (db->dense ? index_bytes(db->dense) : sparse_bytes(db->sparse)));
}

static int32_t sync_meta(gorse_b200_vecdb *db)
{
    const int64_t n = (int64_t)db->ts.size();
    if (!db->meta_dirty) return GORSE_B200_OK;
    cudaStream_t s = db->ctx->stream;
    std::vector<uint8_t> blocked((size_t)n);
    for (int64_t i = 0; i < n; i++) blocked[(size_t)i] = db->hidden[(size_t)i] | db->dead[(size_t)i];
    GB_TRY(db->d_blocked.alloc((size_t)n));
    GB_TRY(db->d_allow.alloc((size_t)n));
    GB_TRY(db->d_cat_off.alloc((size_t)n + 1));
    GB_TRY(db->d_cats.alloc(db->cats.size()));
    if (n) GB_CUDA(cudaMemcpyAsync(db->d_blocked.p, blocked.data(), (size_t)n, cudaMemcpyHostToDevice, s));
    GB_CUDA(cudaMemcpyAsync(db->d_cat_off.p, db->cat_off.data(), sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, s));
    if (!db->cats.empty()) GB_CUDA(cudaMemcpyAsync(db->d_cats.p, db->cats.data(), sizeof(int32_t) * db->cats.size(), cudaMemcpyHostToDevice, s));
    GB_CUDA(cudaStreamSynchronize(s));
    db->meta_dirty = false;
    return GORSE_B200_OK;
}

int32_t vecdb_live_scan(gorse_b200_vecdb *db, DevBuf<int64_t> &scan, int64_t *new_slot)
{
    gorse_b200_ctx *c = db->ctx;
    const int64_t n = (int64_t)db->ts.size();
    DevBuf<uint8_t> d_dead, tmp;
    StreamSync sync{c->stream};
    GB_TRY(d_dead.alloc((size_t)n));
    GB_TRY(scan.alloc((size_t)n + 1));
    size_t tmp_bytes = 0;
    cudaError_t e = n ? cudaMemcpyAsync(d_dead.p, db->dead.data(), (size_t)n, cudaMemcpyHostToDevice, c->stream) : cudaSuccess;
    if (e == cudaSuccess) {
        vecdb_live_kernel<<<div_up(n + 1, 256), 256, 0, c->stream>>>(d_dead.p, n, scan.p);
        c->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, scan.p, n + 1, c->stream);
    if (e != cudaSuccess) { set_error("live scan: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    GB_TRY(tmp.alloc(tmp_bytes));
    e = cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, scan.p, n + 1, c->stream);
    if (e == cudaSuccess && new_slot) e = cudaMemcpyAsync(new_slot, scan.p, sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("live scan: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    return GORSE_B200_OK;
}

int32_t vecdb_allow(gorse_b200_vecdb *db, const int32_t *categories, int32_t n_categories)
{
    gorse_b200_ctx *c = db->ctx;
    const int64_t n = (int64_t)db->ts.size();
    GB_TRY(sync_meta(db));
    if (n_categories) {
        GB_TRY(db->d_want.alloc((size_t)n_categories));
        GB_CUDA(cudaMemcpyAsync(db->d_want.p, categories, sizeof(int32_t) * (size_t)n_categories, cudaMemcpyHostToDevice, c->stream));
    }
    vecdb_allow_kernel<<<div_up(n, 256), 256, 0, c->stream>>>(db->d_blocked.p, db->d_cat_off.p, db->d_cats.p, db->d_want.p, n_categories, n, db->d_allow.p);
    GB_LAUNCHED(c);
    return GORSE_B200_OK;
}

}  // namespace gb

using namespace gb;

extern "C" {

int32_t gorse_b200_vecdb_create(gorse_b200_ctx *ctx, int32_t dim, int32_t distance, gorse_b200_vecdb **out)
{
    GB_CHECK_ARG(ctx != nullptr && out != nullptr, "NULL ctx/out");
    *out = nullptr;
    GB_CHECK_ARG(dim >= 0 && dim <= 16384, "invalid vector dimension %d", dim);
    GB_CHECK_ARG(distance == GORSE_B200_DISTANCE_EUCLIDEAN || distance == GORSE_B200_DISTANCE_DOT || distance == GORSE_B200_DISTANCE_COSINE,
                 "unknown distance %d", distance);
    if (dim == 0 && distance != GORSE_B200_DISTANCE_DOT) {
        set_error("distance method for sparse vector not supported");   // xvec.go:243-245
        return GORSE_B200_ERR_UNSUPPORTED;
    }
    gorse_b200_vecdb *db = new (std::nothrow) gorse_b200_vecdb();
    if (!db) { set_error("host allocation failed"); return GORSE_B200_ERR_OOM; }
    db->ctx = ctx; db->dim = dim; db->distance = distance;
    const int32_t metric = distance == GORSE_B200_DISTANCE_DOT ? GORSE_B200_METRIC_NEG_DOT
                           : distance == GORSE_B200_DISTANCE_EUCLIDEAN ? GORSE_B200_METRIC_EUCLIDEAN : GORSE_B200_METRIC_COSINE;
    int32_t st = dim > 0 ? gorse_b200_index_create(ctx, dim, metric, &db->dense)
                         : gorse_b200_sparse_index_create(ctx, &db->sparse);
    if (st) { delete db; return st; }
    if (db->dense) db->dense->value_bytes = 2;   // bf16 rows until a value that is not bf16-exact arrives (topk.cuh)
    *out = db;
    return GORSE_B200_OK;
}

int32_t gorse_b200_vecdb_destroy(gorse_b200_vecdb *db)
{
    if (!db) return GORSE_B200_OK;
    ScopedDevice sd(db->ctx->device);
    cudaStreamSynchronize(db->ctx->stream);
    gorse_b200_index_destroy(db->dense);
    gorse_b200_sparse_index_destroy(db->sparse);
    delete db;
    return GORSE_B200_OK;
}

int32_t gorse_b200_vecdb_count(gorse_b200_vecdb *db, int64_t *live_out, int64_t *slots_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    if (live_out) *live_out = db->live;
    if (slots_out) *slots_out = (int64_t)db->ts.size();
    return GORSE_B200_OK;
}

int32_t gorse_b200_vecdb_add(gorse_b200_vecdb *db, int64_t n, const float *values, const int64_t *sp_off, const uint32_t *sp_indices,
                             const uint8_t *hidden, const int64_t *timestamp_ms, const int64_t *cat_off, const int32_t *cats,
                             const int64_t *replace, int64_t *first_slot_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    GB_CHECK_ARG(n >= 0, "negative n");
    std::lock_guard<std::mutex> lk(db->mu);
    const int64_t first = (int64_t)db->ts.size();
    if (first_slot_out) *first_slot_out = first;
    if (n == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(values != nullptr || (db->dim == 0 && sp_off && sp_off[n] == 0), "values is NULL");
    GB_CHECK_ARG(db->dim > 0 || sp_off != nullptr, "a sparse collection needs sp_off / sp_indices");
    GB_CHECK_ARG(cat_off == nullptr || cat_off[0] == 0, "cat_off[0] must be 0");
    for (int64_t i = 0; i < n; i++) {
        GB_CHECK_ARG(cat_off == nullptr || cat_off[i + 1] >= cat_off[i], "cat_off not non-decreasing at %lld", (long long)i);
        GB_CHECK_ARG(replace == nullptr || replace[i] < first, "replace[%lld] = %lld is not an existing slot", (long long)i, (long long)replace[i]);
    }
    GB_CHECK_ARG(cat_off == nullptr || cat_off[n] == 0 || cats != nullptr, "cats is NULL");
    int64_t cnt = 0;
    int32_t st = db->dim > 0 ? gorse_b200_index_add(db->dense, values, n, &cnt)
                             : gorse_b200_sparse_index_add(db->sparse, sp_off, sp_indices, values, n, &cnt);
    if (st) return st;
    for (int64_t i = 0; i < n; i++) {
        db->hidden.push_back(hidden ? (hidden[i] != 0) : 0);
        db->dead.push_back(0);
        db->ts.push_back(timestamp_ms ? timestamp_ms[i] : 0);
        if (cat_off) db->cats.insert(db->cats.end(), cats + cat_off[i], cats + cat_off[i + 1]);
        db->cat_off.push_back((int64_t)db->cats.size());
        db->live++;
        if (replace && replace[i] >= 0 && !db->dead[(size_t)replace[i]]) {   // upsert: the old version disappears
            db->dead[(size_t)replace[i]] = 1;
            db->live--;
        }
    }
    db->meta_dirty = true;
    db->gen++;
    return GORSE_B200_OK;
}

// updateItemToItem / updateUserToUser (master/tasks.go:783-877) for the sparse types: the vectors of appendSparseVector
// (logics/vector_writer.go:192-209) built from id rows on the device (sparse_idf_rows) and appended to the index without a host
// rebuild (sparse_append).  Checks that need the ids run on the device into staging buffers; the collection changes after the
// last check has passed.
int32_t gorse_b200_vecdb_add_idf_vectors(gorse_b200_vecdb *db, int64_t n, const int64_t *a_off, const int32_t *a_ids, const float *a_idf,
                                         int32_t a_n_idf, uint32_t a_offset, const int64_t *b_off, const int32_t *b_ids, const float *b_idf,
                                         int32_t b_n_idf, uint32_t b_offset, const uint8_t *hidden, int64_t timestamp_ms, const int64_t *cat_off,
                                         const int32_t *cats, const int64_t *replace, int64_t *slot_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    GB_CHECK_ARG(db->dim == 0, "not a sparse collection");
    GB_CHECK_ARG(n >= 0, "negative n");
    if (n == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(slot_out != nullptr, "slot_out is NULL");
    GB_CHECK_ARG(a_off != nullptr && a_off[0] == 0, "a_off is NULL or a_off[0] != 0");
    GB_CHECK_ARG(b_off == nullptr || b_off[0] == 0, "b_off[0] != 0");
    GB_CHECK_ARG(cat_off == nullptr || cat_off[0] == 0, "cat_off[0] must be 0");
    for (int64_t i = 0; i < n; i++) {
        GB_CHECK_ARG(a_off[i + 1] >= a_off[i], "a_off decreases at row %lld", (long long)i);
        GB_CHECK_ARG(b_off == nullptr || b_off[i + 1] >= b_off[i], "b_off decreases at row %lld", (long long)i);
        GB_CHECK_ARG(cat_off == nullptr || cat_off[i + 1] >= cat_off[i], "cat_off not non-decreasing at %lld", (long long)i);
    }
    GB_CHECK_ARG(a_off[n] == 0 || a_ids != nullptr, "a_ids is NULL");
    GB_CHECK_ARG(a_n_idf >= 0 && (a_n_idf == 0 || a_idf != nullptr), "bad a_idf");
    GB_CHECK_ARG(b_off == nullptr || b_off[n] == 0 || b_ids != nullptr, "b_ids is NULL");
    GB_CHECK_ARG(b_off == nullptr || (b_n_idf >= 0 && (b_n_idf == 0 || b_idf != nullptr)), "bad b_idf");
    GB_CHECK_ARG(cat_off == nullptr || cat_off[n] == 0 || cats != nullptr, "cats is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    std::lock_guard<std::mutex> lk2(db->sparse->mu);
    ScopedDevice sd(db->ctx->device);
    SparseRows rows;
    GB_TRY(sparse_idf_rows(db->ctx, n, a_off, a_ids, a_idf, a_n_idf, a_offset, b_off, b_ids, b_idf, b_n_idf, b_offset, rows));
    // an empty vector is not added (VectorWriter.Add, logics/vector_writer.go:84-92)
    const int64_t first = (int64_t)db->ts.size();
    std::vector<int64_t> slot((size_t)n);
    int64_t added = 0;
    for (int64_t i = 0; i < n; i++) {
        const bool add = rows.row_off[(size_t)i + 1] > rows.row_off[(size_t)i];
        slot[(size_t)i] = add ? first + added++ : -1;
        if (add && replace && replace[i] >= first) {
            set_error("replace[%lld] = %lld is not an existing slot", (long long)i, (long long)replace[i]);
            return GORSE_B200_ERR_ARG;
        }
    }
    GB_TRY(sparse_append(db->sparse, rows));
    for (int64_t i = 0; i < n; i++) {
        slot_out[i] = slot[(size_t)i];
        if (slot[(size_t)i] < 0) continue;
        db->hidden.push_back(hidden ? (hidden[i] != 0) : 0);
        db->dead.push_back(0);
        db->ts.push_back(timestamp_ms);
        if (cat_off) db->cats.insert(db->cats.end(), cats + cat_off[i], cats + cat_off[i + 1]);
        db->cat_off.push_back((int64_t)db->cats.size());
        db->live++;
        if (replace && replace[i] >= 0 && !db->dead[(size_t)replace[i]]) {   // upsert: the old version disappears
            db->dead[(size_t)replace[i]] = 1;
            db->live--;
        }
    }
    if (added) {
        db->meta_dirty = true;
        db->gen++;
    }
    return GORSE_B200_OK;
}

int32_t gorse_b200_vecdb_get(gorse_b200_vecdb *db, const int64_t *slots, int64_t n, float *values_out, uint8_t *hidden_out,
                             int64_t *timestamp_out, uint8_t *live_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    GB_CHECK_ARG(n >= 0 && (n == 0 || slots != nullptr), "bad slots");
    std::lock_guard<std::mutex> lk(db->mu);
    const int64_t total = (int64_t)db->ts.size();
    ScopedDevice sd(db->ctx->device);
    std::vector<int64_t> rows(values_out && db->dim > 0 ? (size_t)n : 0);   // the stored row of each entry, -1 for none
    for (int64_t i = 0; i < n; i++) {
        const int64_t s = slots[i];
        const bool ok = s >= 0 && s < total && !db->dead[(size_t)s];
        if (live_out) live_out[i] = ok;
        if (hidden_out) hidden_out[i] = ok ? db->hidden[(size_t)s] : 0;
        if (timestamp_out) timestamp_out[i] = ok ? db->ts[(size_t)s] : 0;
        if (!rows.empty()) {
            rows[(size_t)i] = ok ? s : -1;
            if (!ok) memset(values_out + i * db->dim, 0, sizeof(float) * db->dim);
        }
    }
    if (rows.empty()) return GORSE_B200_OK;
    return index_download_rows(db->dense, rows.data(), n, values_out);
}

int32_t gorse_b200_vecdb_get_sparse(gorse_b200_vecdb *db, int64_t slot, uint32_t *indices_out, float *values_out, int32_t cap, int32_t *nnz_out)
{
    GB_CHECK_ARG(db != nullptr && nnz_out != nullptr, "NULL argument");
    GB_CHECK_ARG(db->dim == 0, "not a sparse collection");
    std::lock_guard<std::mutex> lk(db->mu);
    GB_CHECK_ARG(slot >= 0 && slot < (int64_t)db->ts.size(), "slot out of range");
    const int64_t b = db->sparse->h_off[(size_t)slot], e = db->sparse->h_off[(size_t)slot + 1];
    *nnz_out = (int32_t)(e - b);
    for (int64_t t = b; t < e && t - b < cap; t++) {
        if (indices_out) indices_out[t - b] = db->sparse->h_ind[(size_t)t];
        if (values_out) values_out[t - b] = db->sparse->h_val[(size_t)t];
    }
    return GORSE_B200_OK;
}

int32_t gorse_b200_vecdb_delete_before(gorse_b200_vecdb *db, int64_t timestamp_ms, int64_t *slots_out, int64_t cap, int64_t *count_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    int64_t cnt = 0;
    for (size_t i = 0; i < db->ts.size(); i++)
        if (!db->dead[i] && db->ts[i] < timestamp_ms) {   // "timestamp < t", xvec.go:370
            db->dead[i] = 1;
            db->live--;
            if (slots_out && cnt < cap) slots_out[cnt] = (int64_t)i;
            cnt++;
        }
    if (cnt) {
        db->meta_dirty = true;
        db->gen++;
    }
    if (count_out) *count_out = cnt;
    return GORSE_B200_OK;
}

// Optimize (storage/vectors/database.go:109; xvec.go:125-131).  The live flags are scanned on the device; the scan is the
// renumbering, which the index applies to its own rows (index_compact, sparse_compact) and the host applies to the metadata.
// Every new buffer, device or host, exists before anything of the collection changes.
int32_t gorse_b200_vecdb_compact(gorse_b200_vecdb *db, int64_t *new_slot_out, int64_t *bytes_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    std::lock_guard<std::mutex> lk2(db->dense ? db->dense->mu : db->sparse->mu);
    const int64_t n = (int64_t)db->ts.size(), live = db->live;
    if (bytes_out) bytes_out[0] = bytes_out[1] = vecdb_bytes(db);
    if (live == n) {   // nothing to reclaim
        if (new_slot_out)
            for (int64_t s = 0; s < n; s++) new_slot_out[s] = s;
        return GORSE_B200_OK;
    }
    gorse_b200_ctx *c = db->ctx;
    ScopedDevice sd(c->device);
    std::vector<int64_t> new_slot((size_t)n + 1);
    DevBuf<int64_t> scan;
    StreamSync sync{c->stream};
    GB_TRY(vecdb_live_scan(db, scan, new_slot.data()));
    // the compacted host metadata
    std::vector<uint8_t> hidden((size_t)live), dead((size_t)live, 0);
    std::vector<int64_t> ts((size_t)live), cat_off((size_t)live + 1, 0);
    std::vector<int32_t> cats;
    cats.reserve(db->cats.size());
    for (int64_t s = 0; s < n; s++) {
        if (db->dead[(size_t)s]) continue;
        const size_t to = (size_t)new_slot[(size_t)s];
        hidden[to] = db->hidden[(size_t)s];
        ts[to] = db->ts[(size_t)s];
        cats.insert(cats.end(), db->cats.begin() + db->cat_off[(size_t)s], db->cats.begin() + db->cat_off[(size_t)s + 1]);
        cat_off[to + 1] = (int64_t)cats.size();
    }
    GB_TRY(db->dense ? index_compact(db->dense, scan.p, live) : sparse_compact(db->sparse, scan.p, live));
    db->hidden.swap(hidden); db->dead.swap(dead); db->ts.swap(ts); db->cat_off.swap(cat_off); db->cats.swap(cats);
    db->meta_dirty = true;
    db->gen++;
    // every device buffer whose size follows the slot count; the next call that needs one allocates (and zeroes) it again
    db->d_blocked.free(); db->d_allow.free(); db->d_cat_off.free(); db->d_cats.free();
    db->stage.acc.free(); db->stage.seen.free(); db->stage.uacc.free(); db->stage.flag.free(); db->stage.touched.free(); db->stage.item_ok.free();
    if (new_slot_out)   // `dead` holds the old flags after the swap
        for (int64_t s = 0; s < n; s++) new_slot_out[s] = dead[(size_t)s] ? -1 : new_slot[(size_t)s];
    if (bytes_out) bytes_out[1] = vecdb_bytes(db);
    return GORSE_B200_OK;
}

int32_t gorse_b200_vecdb_storage(gorse_b200_vecdb *db, int32_t *value_bytes_out, int64_t *device_bytes_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    std::lock_guard<std::mutex> lk(db->mu);
    std::lock_guard<std::mutex> lk2(db->dense ? db->dense->mu : db->sparse->mu);
    if (value_bytes_out) *value_bytes_out = db->dense ? db->dense->value_bytes : 0;
    if (device_bytes_out) *device_bytes_out = vecdb_bytes(db);
    return GORSE_B200_OK;
}

int32_t gorse_b200_vecdb_query(gorse_b200_vecdb *db, int64_t nq, const float *q_values, const int64_t *q_sp_off, const uint32_t *q_sp_indices,
                               const int32_t *categories, int32_t n_categories, int32_t topk, int64_t *slots_out, float *scores_out,
                               int32_t *count_out)
{
    GB_CHECK_ARG(db != nullptr, "collection is NULL");
    GB_CHECK_ARG(nq >= 0 && n_categories >= 0, "negative count");
    if (nq == 0) return GORSE_B200_OK;
    GB_CHECK_ARG(count_out != nullptr, "count_out is NULL");
    if (topk <= 0) {   // xvec.go:374-376
        for (int64_t q = 0; q < nq; q++) count_out[q] = 0;
        return GORSE_B200_OK;
    }
    GB_CHECK_ARG(slots_out != nullptr && scores_out != nullptr, "NULL output");
    GB_CHECK_ARG(n_categories == 0 || categories != nullptr, "categories is NULL");
    GB_CHECK_ARG(db->dim == 0 || q_values != nullptr, "q_values is NULL");
    GB_CHECK_ARG(db->dim > 0 || q_sp_off != nullptr, "a sparse collection is queried with q_sp_off / q_sp_indices");
    std::lock_guard<std::mutex> lk(db->mu);
    const int64_t n = (int64_t)db->ts.size();
    gorse_b200_ctx *c = db->ctx;
    ScopedDevice sd(c->device);
    if (n == 0) {
        for (int64_t q = 0; q < nq; q++) count_out[q] = 0;
        return GORSE_B200_OK;
    }
    GB_TRY(vecdb_allow(db, categories, n_categories));
    if (db->dim > 0) {   // the pipeline's score is the negated distance of the index (-dot / Euclidean): xvec.go:425-427, Dot -> dot
        std::lock_guard<std::mutex> lk2(db->dense->mu);
        return recall::recall_rows(db->dense, db->d_allow.p, nq, q_values, nullptr, topk, nullptr, nullptr, nullptr, nullptr, slots_out, scores_out,
                                   count_out, nullptr);   // no exclusions: row q at q * topk
    }
    for (int64_t q = 0; q < nq; q++)
        for (int64_t t = q_sp_off[q]; t < q_sp_off[q + 1]; t++)
            GB_CHECK_ARG(t == q_sp_off[q] || q_sp_indices[t] > q_sp_indices[t - 1], "query %lld: indices not strictly ascending", (long long)q);
    // no answer is longer than the collection: the search answers kc columns, the rest of each row is padding
    const int32_t kc = (int32_t)std::min<int64_t>(topk, n);
    std::vector<int32_t> idx((size_t)nq * kc);
    std::vector<float> dot(kc < topk ? (size_t)nq * kc : 0);
    {
        std::lock_guard<std::mutex> lk2(db->sparse->mu);
        GB_TRY(sparse_search_host(db->sparse, 0, nq, q_sp_off, q_sp_indices, q_values, db->d_allow.p, kc, idx.data(), kc < topk ? dot.data() : scores_out,
                                  count_out));
    }
    for (int64_t q = 0; q < nq; q++)
        for (int64_t t = 0; t < topk; t++) {
            slots_out[q * topk + t] = t < kc ? idx[(size_t)(q * kc + t)] : -1;
            if (kc < topk) scores_out[q * topk + t] = t < kc ? dot[(size_t)(q * kc + t)] : 0.f;
        }
    return GORSE_B200_OK;
}

// master/tasks.go:925-961: after Fit the item factors of the predictable items become the "collaborative_filtering_<id>"
// collection (distance Dot).  The reference walks GetItemFactor(i) row by row into []vectors.Vector batches; here the rows go
// from the model's item table to the collection device to device.  slot_of_item_out[n_items]: the slot of each item, -1 for
// items without training feedback (they are skipped, :943).  Single-GPU models (the replicated Q of a distributed model is
// complete on every rank, but predictability needs all ranks' rows).
int32_t gorse_b200_vecdb_add_item_factors(gorse_b200_vecdb *db, gorse_b200_cf *cf, const uint8_t *hidden, int64_t timestamp_ms,
                                          const int64_t *cat_off, const int32_t *cats, int64_t *slot_of_item_out)
{
    GB_CHECK_ARG(db != nullptr && cf != nullptr, "NULL collection / model");
    GB_CHECK_ARG(db->dim == cf->d, "collection dimension %d != model factors %d", db->dim, cf->d);
    GB_CHECK_ARG(cf->ctx->world == 1, "hand-off from a distributed model is not supported");
    GB_CHECK_ARG(db->ctx->device == cf->ctx->device, "collection and model live on different devices");
    GB_CHECK_ARG(cat_off == nullptr || cat_off[0] == 0, "cat_off[0] must be 0");
    std::lock_guard<std::mutex> lk(db->mu);
    gorse_b200_ctx *c = db->ctx;
    ScopedDevice sd(c->device);
    const int32_t I = cf->n_items;
    std::vector<int32_t> flag((size_t)I), items;
    DevBuf<int32_t> d_flag, d_items;
    StreamSync sync{c->stream};
    GB_TRY(d_flag.alloc((size_t)std::max(I, 1)));
    cudaError_t e = cudaMemsetAsync(d_flag.p, 0, sizeof(int32_t) * (size_t)std::max(I, 1), c->stream);
    if (e == cudaSuccess && cf->n_feedback > 0) {
        vecdb_mark_items_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(cf->user_items.p, cf->n_feedback, d_flag.p);
        c->launches++;
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && I) e = cudaMemcpyAsync(flag.data(), d_flag.p, sizeof(int32_t) * (size_t)I, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("add_item_factors: %s", cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    const int64_t first = (int64_t)db->ts.size();
    for (int32_t i = 0; i < I; i++) {
        if (slot_of_item_out) slot_of_item_out[i] = flag[(size_t)i] ? first + (int64_t)items.size() : -1;
        if (flag[(size_t)i]) items.push_back(i);
    }
    const int64_t n = (int64_t)items.size();
    if (n == 0) return GORSE_B200_OK;
    gorse_b200_index *ix = db->dense;
    {   // the factor rows go device to device; a bf16 collection checks them there and promotes when one is not bf16-exact
        std::lock_guard<std::mutex> lk2(ix->mu);
        GB_TRY(d_items.upload(items.data(), (size_t)n, c->stream));
        GB_TRY(index_append(ix, cf->Q.p, d_items.p, n, false));
    }
    for (int64_t s2 = 0; s2 < n; s2++) {
        const int32_t it = items[(size_t)s2];
        db->hidden.push_back(hidden ? (hidden[it] != 0) : 0);
        db->dead.push_back(0);
        db->ts.push_back(timestamp_ms);
        if (cat_off) db->cats.insert(db->cats.end(), cats + cat_off[it], cats + cat_off[it + 1]);
        db->cat_off.push_back((int64_t)db->cats.size());
        db->live++;
    }
    db->meta_dirty = true;
    db->gen++;
    return GORSE_B200_OK;
}

}  // extern "C"
