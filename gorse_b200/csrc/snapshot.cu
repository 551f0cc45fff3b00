// snapshot.cu -- a vector collection written as a byte stream (gorse_b200_vecdb_save) and rebuilt from one on any context
// (gorse_b200_vecdb_load): what lets a worker, a server or a restarted master hold the collections the master built, as the
// reference's default backend reopens its collections from disk in Init (storage/vectors/xvec.go:60-123).  The stream format
// is documented in include/gorse_b200.h.
//
// Dense rows never pass through a host copy of the collection: save gathers each chunk's live rows on the device (the live-slot
// scan of compaction names them) and downloads it on the copy stream into one of two pinned staging buffers while the callback
// writes the other; load fills one pinned buffer from the callback while the other is copied into the index's rows.  The
// metadata and the sparse rows are host state of the collection already; they stream through the same staging buffer.
#include <algorithm>
#include <cmath>

#include "sparse.cuh"
#include "vecdb.cuh"

namespace gb {
namespace {

constexpr char MAGIC[8] = {'G', 'B', '2', '0', '0', 'V', 'D', 'B'};
constexpr uint32_t VERSION = 1;
constexpr int64_t STAGE_BYTES = 64ll << 20;   // each of the two staging buffers, at most
constexpr int64_t MIN_STAGE_BYTES = 64ll << 10;   // one row of the widest dense collection (16384 fp32)

struct Header {
    char magic[8];
    uint32_t version;
    int32_t dim, distance;
    uint32_t reserved;
    int64_t n, nnz, n_cats;
};
static_assert(sizeof(Header) == 48, "the stream header is 48 bytes without padding");

// out[(j - j0) * d ..] = X[slot(j) * d ..] for the live rows j in [j0, j0 + m): slot(j) is the slot whose scan entry is j and
// whose successor's is j + 1, found by a binary search of scan[0 .. n] (scan[n] = the live count).  One warp per row;
// V = float4 when d % 4 == 0 (dv = d / 4), else float (dv = d); bf16 rows (V = uint2 / uint16_t) are widened to W on the way.
template <typename V, typename W>
__global__ void snapshot_gather_kernel(const V *X, int dv, const int64_t *scan, int64_t n, int64_t j0, int64_t m, W *out)
{
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < m; r += nw) {
        const int64_t j = j0 + r;
        int64_t lo = 0, hi = n;   // scan[lo] <= j < scan[hi]
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg(scan + mid) <= j) lo = mid;
            else hi = mid;
        }
        const V *src = X + lo * dv;
        W *dst = out + r * dv;
        for (int c = lane; c < dv; c += 32) dst[c] = widen(src[c]);
    }
}

// the two pinned staging buffers, the device gather buffers and their events; `sync`, declared last and so destroyed first,
// drains both streams before any of them is freed
struct Staging {
    gorse_b200_ctx *c;
    PinnedBuf<char> h[2];
    DevBuf<float> d[2];
    Event gathered[2], copied[2];
    PinnedBuf<int32_t> flag;   // [2]: load's inexact flag of the chunk in each buffer
    StreamSync sync;
    explicit Staging(gorse_b200_ctx *ctx) : c(ctx), sync{ctx->stream, ctx->copy_stream} {}
    int32_t alloc(int64_t bytes, int buffers, bool device)
    {
        for (int b = 0; b < buffers; b++) {
            GB_TRY(h[b].alloc((size_t)bytes));
            GB_TRY(copied[b].create());
            if (!device) continue;
            GB_TRY(d[b].alloc((size_t)bytes / sizeof(float)));
            GB_TRY(gathered[b].create());
        }
        if (device) {
            GB_TRY(flag.alloc(2));
            flag.p[0] = flag.p[1] = 0;   // pinned memory comes back uninitialised
        }
        return GORSE_B200_OK;
    }
    // a load's chunk k fills h[k & 1]: wait_free waits until chunk k - 2's upload from it has finished, and in_flight marks
    // it busy again once chunk k's upload is queued on the copy stream
    cudaError_t wait_free(int64_t k) { return k >= 2 ? cudaEventSynchronize(copied[k & 1].e) : cudaSuccess; }
    cudaError_t in_flight(int64_t k) { return cudaEventRecord(copied[k & 1].e, c->copy_stream); }
};

// the caller's write callback behind a staging buffer: put() appends and hands full buffers on, direct() hands a buffer of the
// caller's on after the pending bytes
struct Writer {
    gorse_b200_write_fn fn;
    void *user;
    char *buf;
    int64_t cap, used = 0, pos = 0;   // pos: bytes handed to the callback
    const char *who = "snapshot save";
    int32_t direct(const void *p, int64_t bytes)
    {
        if (bytes == 0) return GORSE_B200_OK;
        if (fn(user, p, bytes) != 0) {
            set_error("%s: the write callback failed at byte %lld", who, (long long)pos);
            return GORSE_B200_ERR_IO;
        }
        pos += bytes;
        return GORSE_B200_OK;
    }
    int32_t flush()
    {
        const int64_t m = used;
        used = 0;
        return direct(buf, m);
    }
    int32_t put(const void *src, int64_t bytes)
    {
        const char *s = static_cast<const char *>(src);
        while (bytes > 0) {
            const int64_t m = std::min(bytes, cap - used);
            memcpy(buf + used, s, (size_t)m);
            used += m; s += m; bytes -= m;
            if (used == cap) GB_TRY(flush());
        }
        return GORSE_B200_OK;
    }
};

// A save's chunks 0 .. chunks - 1 through the staging buffers: gather(k, d) launches chunk k's gather into the device buffer d
// on the context's stream, and bytes(k) is the chunk's length.  Chunk k is downloaded into h[k & 1] on the copy stream and
// written while chunk k + 1 is gathered and downloaded; chunk k + 2 reuses the buffers once chunk k is written.
template <typename Bytes, typename Gather>
int32_t write_chunks(Staging &stg, Writer &w, int64_t chunks, Bytes bytes, Gather gather)
{
    gorse_b200_ctx *c = stg.c;
    auto enqueue = [&](int64_t k) {
        const int b = (int)(k & 1);
        gather(k, stg.d[b].p);
        c->launches++;
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaEventRecord(stg.gathered[b].e, c->stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(c->copy_stream, stg.gathered[b].e, 0);
        if (e == cudaSuccess) e = cudaMemcpyAsync(stg.h[b].p, stg.d[b].p, (size_t)bytes(k), cudaMemcpyDeviceToHost, c->copy_stream);
        if (e == cudaSuccess) e = cudaEventRecord(stg.copied[b].e, c->copy_stream);
        return e;
    };
    cudaError_t e = cudaSuccess;
    int32_t st = GORSE_B200_OK;
    for (int64_t k = 0; k < std::min<int64_t>(2, chunks) && e == cudaSuccess; k++) e = enqueue(k);
    for (int64_t k = 0; k < chunks && e == cudaSuccess && st == GORSE_B200_OK; k++) {
        const int b = (int)(k & 1);
        e = cudaEventSynchronize(stg.copied[b].e);
        if (e == cudaSuccess) st = w.direct(stg.h[b].p, bytes(k));
        if (e == cudaSuccess && st == GORSE_B200_OK && k + 2 < chunks) e = enqueue(k + 2);
    }
    cudaStreamSynchronize(c->copy_stream);
    if (e != cudaSuccess) { set_error("%s: %s", w.who, cudaGetErrorString(e)); return GORSE_B200_ERR_CUDA; }
    return st;
}

// the caller's read callback: get() reads exactly `bytes` or fails, naming the field and its byte offset
struct Reader {
    gorse_b200_read_fn fn;
    void *user;
    int64_t pos = 0;   // bytes read
    const char *who = "snapshot load";
    int32_t get(void *dst, int64_t bytes, const char *field)
    {
        char *d = static_cast<char *>(dst);
        while (bytes > 0) {
            const int64_t r = fn(user, d, bytes);
            if (r < 0 || r > bytes) {
                set_error("%s: the read callback failed at byte %lld (%s)", who, (long long)pos, field);
                return GORSE_B200_ERR_IO;
            }
            if (r == 0) {
                set_error("%s: the stream ends at byte %lld, inside %s", who, (long long)pos, field);
                return GORSE_B200_ERR_ARG;
            }
            d += r; bytes -= r; pos += r;
        }
        return GORSE_B200_OK;
    }
    // ERR_ARG for a field that fails its check, naming the field and its byte offset
    int32_t bad(const char *field, int64_t at, const char *what) const
    {
        set_error("%s: bad %s at byte %lld: %s", who, field, (long long)at, what);
        return GORSE_B200_ERR_ARG;
    }
    // count elements into v, grown piece by piece: a header that claims more than the stream holds allocates no more than arrived
    template <typename T>
    int32_t array(std::vector<T> &v, int64_t count, const char *field)
    {
        constexpr int64_t PIECE = (4ll << 20) / (int64_t)sizeof(T);
        v.clear();
        for (int64_t i = 0; i < count; i += PIECE) {
            const int64_t m = std::min(PIECE, count - i);
            v.resize((size_t)(i + m));
            GB_TRY(get(v.data() + i, m * (int64_t)sizeof(T), field));
        }
        return GORSE_B200_OK;
    }
};

// a field read through Reader r that fails cond ends the call with r.bad(field, at, what)
#define STREAM_CHECK(r, cond, field, at, what)          \
    do {                                                \
        if (!(cond)) return (r).bad(field, at, what);   \
    } while (0)

// offsets[n + 1] of a section starting at byte `at`: from 0, never decreasing, ending at `total`
int32_t check_offsets(const Reader &r, const std::vector<int64_t> &off, int64_t total, const char *field, int64_t at)
{
    STREAM_CHECK(r, off[0] == 0, field, at, "the first offset is not 0");
    const int64_t n = (int64_t)off.size() - 1;
    for (int64_t i = 0; i < n; i++) STREAM_CHECK(r, off[(size_t)i + 1] >= off[(size_t)i], field, at + 8 * (i + 1), "offsets decrease");
    STREAM_CHECK(r, off[(size_t)n] == total, field, at + 8 * n, "the last offset disagrees with the header's count");
    return GORSE_B200_OK;
}

int32_t save(gorse_b200_vecdb *db, gorse_b200_write_fn write, void *user, int64_t *new_slot_out, int64_t *bytes_out)
{
    std::lock_guard<std::mutex> lk(db->mu);
    std::lock_guard<std::mutex> lk2(db->dense ? db->dense->mu : db->sparse->mu);
    gorse_b200_ctx *c = db->ctx;
    ScopedDevice sd(c->device);
    const int64_t n = (int64_t)db->ts.size(), live = db->live, dim = db->dim;
    const gorse_b200_sparse_index *sx = db->sparse;
    Header h{};
    memcpy(h.magic, MAGIC, sizeof(MAGIC));
    h.version = VERSION;
    h.dim = db->dim;
    h.distance = db->distance;
    h.n = live;
    for (int64_t s = 0; s < n; s++) {
        if (db->dead[(size_t)s]) continue;
        h.n_cats += db->cat_off[(size_t)s + 1] - db->cat_off[(size_t)s];
        if (sx) h.nnz += sx->h_off[(size_t)s + 1] - sx->h_off[(size_t)s];
    }
    const int64_t values = dim > 0 ? 4 * live * dim : 8 * (live + 1) + 8 * h.nnz;
    const int64_t total = (int64_t)sizeof(Header) + 17 * live + 8 + 4 * h.n_cats + values;
    Staging stg(c);
    const int64_t cap = std::min(STAGE_BYTES, std::max(MIN_STAGE_BYTES, total));
    GB_TRY(stg.alloc(cap, dim > 0 && live > 0 ? 2 : 1, dim > 0 && live > 0));
    Writer w{write, user, stg.h[0].p, cap};
    GB_TRY(w.put(&h, sizeof(h)));
    for (int64_t s = 0; s < n; s++)
        if (!db->dead[(size_t)s]) GB_TRY(w.put(&db->hidden[(size_t)s], 1));
    for (int64_t s = 0; s < n; s++)
        if (!db->dead[(size_t)s]) GB_TRY(w.put(&db->ts[(size_t)s], 8));
    int64_t o = 0;
    GB_TRY(w.put(&o, 8));
    for (int64_t s = 0; s < n; s++)
        if (!db->dead[(size_t)s]) {
            o += db->cat_off[(size_t)s + 1] - db->cat_off[(size_t)s];
            GB_TRY(w.put(&o, 8));
        }
    for (int64_t s = 0; s < n; s++)
        if (!db->dead[(size_t)s])
            GB_TRY(w.put(db->cats.data() + db->cat_off[(size_t)s], 4 * (db->cat_off[(size_t)s + 1] - db->cat_off[(size_t)s])));
    if (sx) {
        o = 0;
        GB_TRY(w.put(&o, 8));
        for (int64_t s = 0; s < n; s++)
            if (!db->dead[(size_t)s]) {
                o += sx->h_off[(size_t)s + 1] - sx->h_off[(size_t)s];
                GB_TRY(w.put(&o, 8));
            }
        for (int64_t s = 0; s < n; s++)
            if (!db->dead[(size_t)s]) GB_TRY(w.put(sx->h_ind.data() + sx->h_off[(size_t)s], 4 * (sx->h_off[(size_t)s + 1] - sx->h_off[(size_t)s])));
        for (int64_t s = 0; s < n; s++)
            if (!db->dead[(size_t)s]) GB_TRY(w.put(sx->h_val.data() + sx->h_off[(size_t)s], 4 * (sx->h_off[(size_t)s + 1] - sx->h_off[(size_t)s])));
    }
    GB_TRY(w.flush());
    if (dim > 0 && live > 0) {
        // chunk k = the live rows [k R, k R + R)
        DevBuf<int64_t> scan;
        GB_TRY(vecdb_live_scan(db, scan, nullptr));
        const gorse_b200_index *ix = db->dense;
        const int64_t R = cap / (4 * dim), chunks = (live + R - 1) / R;
        auto rows_of = [&](int64_t k) { return std::min(R, live - k * R); };
        GB_TRY(write_chunks(stg, w, chunks, [&](int64_t k) { return 4 * rows_of(k) * dim; }, [&](int64_t k, float *d) {
            const int64_t m = rows_of(k);
            const unsigned grid = (unsigned)std::min<int64_t>((m + 7) / 8, (int64_t)c->sm_count * 16);
            with_rows(ix->rows(), [&](auto x) {   // the stream holds fp32 values: bf16 rows are widened by the gather
                using Q = typename row_quad_type<row_elem_t<decltype(x)>>::type;
                if (dim % 4 == 0)
                    snapshot_gather_kernel<<<grid, 256, 0, c->stream>>>(reinterpret_cast<const Q *>(x), (int)(dim / 4), scan.p, n, k * R, m,
                                                                       reinterpret_cast<float4 *>(d));
                else
                    snapshot_gather_kernel<<<grid, 256, 0, c->stream>>>(x, (int)dim, scan.p, n, k * R, m, d);
            });
        }));
    }
    if (new_slot_out)
        for (int64_t s = 0, j = 0; s < n; s++) new_slot_out[s] = db->dead[(size_t)s] ? -1 : j++;
    if (bytes_out) *bytes_out = w.pos;
    return GORSE_B200_OK;
}

// the header's fields, each count against the others and against int64 overflow of its section
int32_t check_header(const Reader &r, const Header &h)
{
    STREAM_CHECK(r, memcmp(h.magic, MAGIC, sizeof(MAGIC)) == 0, "magic", 0, "not a gorse_b200 collection stream");
    STREAM_CHECK(r, h.version == VERSION, "version", 8, "unknown version");
    STREAM_CHECK(r, h.dim >= 0 && h.dim <= 16384, "dim", 12, "outside [0, 16384]");
    STREAM_CHECK(r, h.distance == GORSE_B200_DISTANCE_EUCLIDEAN || h.distance == GORSE_B200_DISTANCE_DOT || h.distance == GORSE_B200_DISTANCE_COSINE,
               "distance", 16, "unknown distance");
    STREAM_CHECK(r, h.dim > 0 || h.distance == GORSE_B200_DISTANCE_DOT, "distance", 16, "a sparse collection is Dot");
    STREAM_CHECK(r, h.reserved == 0, "reserved", 20, "not 0");
    // every section's byte count, and their sum, fit in an int64 below 2^62
    constexpr int64_t LIM = 1ll << 62;
    STREAM_CHECK(r, h.n >= 0 && h.n < LIM / 32, "n", 24, "negative or too large");
    STREAM_CHECK(r, h.dim > 0 || h.n < (1ll << 31) - 1, "n", 24, "more than 2^31 - 1 sparse vectors");
    STREAM_CHECK(r, h.dim > 0 || h.n < LIM / 32, "n", 24, "too large");
    STREAM_CHECK(r, h.dim == 0 || h.n <= LIM / 8 / h.dim, "n", 24, "n * dim overflows");
    STREAM_CHECK(r, h.nnz >= 0 && h.nnz < LIM / 16, "nnz", 32, "negative or too large");
    STREAM_CHECK(r, h.dim == 0 || h.nnz == 0, "nnz", 32, "not 0 in a dense collection");
    STREAM_CHECK(r, h.n_cats >= 0 && h.n_cats < LIM / 16, "category count", 40, "negative or too large");
    return GORSE_B200_OK;
}

int32_t load(gorse_b200_ctx *ctx, gorse_b200_read_fn read, void *user, gorse_b200_vecdb **out, int64_t *bytes_out)
{
    Reader r{read, user};
    Header h;
    GB_TRY(r.get(&h, sizeof(h), "header"));
    GB_TRY(check_header(r, h));
    const int64_t n = h.n, dim = h.dim;
    std::vector<uint8_t> hidden;
    std::vector<int64_t> ts, cat_off;
    std::vector<int32_t> cats;
    int64_t at = r.pos;
    GB_TRY(r.array(hidden, n, "hidden"));
    for (int64_t i = 0; i < n; i++) STREAM_CHECK(r, hidden[(size_t)i] <= 1, "hidden", at + i, "neither 0 nor 1");
    GB_TRY(r.array(ts, n, "timestamp_ms"));
    at = r.pos;
    GB_TRY(r.array(cat_off, n + 1, "cat_off"));
    GB_TRY(check_offsets(r, cat_off, h.n_cats, "cat_off", at));
    GB_TRY(r.array(cats, h.n_cats, "cats"));
    std::vector<int64_t> sp_off;
    std::vector<uint32_t> sp_ind;
    std::vector<float> sp_val;
    uint32_t n_features = 0;
    if (dim == 0) {
        at = r.pos;
        GB_TRY(r.array(sp_off, n + 1, "off"));
        GB_TRY(check_offsets(r, sp_off, h.nnz, "off", at));
        at = r.pos;
        GB_TRY(r.array(sp_ind, h.nnz, "ind"));
        for (int64_t i = 0; i < n; i++)
            for (int64_t t = sp_off[(size_t)i]; t < sp_off[(size_t)i + 1]; t++) {
                STREAM_CHECK(r, t == sp_off[(size_t)i] || sp_ind[(size_t)t] > sp_ind[(size_t)t - 1], "ind", at + 4 * t,
                           "indices of a vector not strictly ascending");
                STREAM_CHECK(r, sp_ind[(size_t)t] < 0x7fffffffu, "ind", at + 4 * t, "index >= 0x7fffffff");
                n_features = std::max(n_features, sp_ind[(size_t)t] + 1);
            }
        at = r.pos;
        GB_TRY(r.array(sp_val, h.nnz, "val"));
        for (int64_t t = 0; t < h.nnz; t++) STREAM_CHECK(r, !std::isnan(sp_val[(size_t)t]), "val", at + 4 * t, "NaN value");
    }
    std::vector<uint8_t> dead((size_t)n, 0);
    // the handle is this call's until it returns: nobody else can take its locks
    gorse_b200_vecdb *db = nullptr;
    GB_TRY(gorse_b200_vecdb_create(ctx, h.dim, h.distance, &db));
    int32_t st = GORSE_B200_OK;
    {
        ScopedDevice sd(ctx->device);
        if (dim == 0) {
            gorse_b200_sparse_index *sx = db->sparse;
            sx->h_off.swap(sp_off); sx->h_ind.swap(sp_ind); sx->h_val.swap(sp_val);
            sx->n_features = n_features;
            sx->dirty = true;
            st = sparse_sync_device(sx);
        } else if (n > 0) {
            // chunk k = rows [k R, k R + R): read into h[k & 1] while chunk k - 1 is copied on the copy stream.  While the
            // collection is bf16 a chunk goes through the device buffer d[k & 1] and is narrowed into the rows there; its inexact
            // flag comes back with it and is read when its buffers are reused (or at the end).  The first chunk k0 that was not
            // bf16-exact promotes the collection: the rows before it are widened, and chunk k0 and the one after it, whose fp32
            // values are still in the device buffers, are copied in; later chunks go straight into the fp32 rows.
            gorse_b200_index *ix = db->dense;
            Staging stg(ctx);
            const int64_t cap = std::min(STAGE_BYTES, std::max(MIN_STAGE_BYTES, 4 * n * dim));
            st = index_reserve(ix, n);
            if (st == GORSE_B200_OK) st = stg.alloc(cap, 2, ix->value_bytes == 2);
            if (st == GORSE_B200_OK) st = ix->inexact.grow(2);
            const int64_t R = cap / (4 * dim), chunks = st ? 0 : (n + R - 1) / R;
            auto rows_of = [&](int64_t k) { return std::min(R, n - k * R); };
            cudaError_t e = cudaSuccess;
            auto promote_at = [&](int64_t k0, int64_t k1) {   // chunks [k0, k1) were narrowed; k0 was not exact
                e = cudaStreamSynchronize(ctx->copy_stream);
                if (e == cudaSuccess) st = index_promote(ix, k0 * R);
                for (int64_t k = k0; k < k1 && e == cudaSuccess && st == GORSE_B200_OK; k++)
                    e = cudaMemcpyAsync(ix->X.p + k * R * dim, stg.d[k & 1].p, sizeof(float) * rows_of(k) * dim, cudaMemcpyDeviceToDevice, ctx->copy_stream);
            };
            for (int64_t k = 0; k < chunks && e == cudaSuccess && st == GORSE_B200_OK; k++) {
                const int b = (int)(k & 1);
                const int64_t j0 = k * R, bytes = 4 * rows_of(k) * dim;
                e = stg.wait_free(k);
                if (e == cudaSuccess && k >= 2 && ix->value_bytes == 2 && stg.flag.p[b]) promote_at(k - 2, k);   // chunk k - 2's flag
                if (e == cudaSuccess && st == GORSE_B200_OK) st = r.get(stg.h[b].p, bytes, "values");
                if (e != cudaSuccess || st != GORSE_B200_OK) break;
                if (ix->value_bytes == 2) {
                    e = cudaMemcpyAsync(stg.d[b].p, stg.h[b].p, (size_t)bytes, cudaMemcpyHostToDevice, ctx->copy_stream);
                    if (e == cudaSuccess) e = cudaMemsetAsync(ix->inexact.p + b, 0, sizeof(int32_t), ctx->copy_stream);
                    if (e == cudaSuccess) e = index_narrow((int)dim, ctx, ctx->copy_stream, stg.d[b].p, nullptr, rows_of(k), ix->Xh.p + j0 * dim, ix->inexact.p + b);
                    if (e == cudaSuccess) e = cudaMemcpyAsync(stg.flag.p + b, ix->inexact.p + b, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->copy_stream);
                } else
                    e = cudaMemcpyAsync(ix->X.p + j0 * dim, stg.h[b].p, (size_t)bytes, cudaMemcpyHostToDevice, ctx->copy_stream);
                if (e == cudaSuccess) e = stg.in_flight(k);
            }
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->copy_stream);
            for (int64_t k = std::max<int64_t>(0, chunks - 2); k < chunks && e == cudaSuccess && st == GORSE_B200_OK; k++)
                if (ix->value_bytes == 2 && stg.flag.p[k & 1]) promote_at(k, chunks);
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->copy_stream);
            if (e != cudaSuccess && st == GORSE_B200_OK) {
                set_error("snapshot load: %s", cudaGetErrorString(e));
                st = e == cudaErrorMemoryAllocation ? GORSE_B200_ERR_OOM : GORSE_B200_ERR_CUDA;
            }
            ix->n = n;
            ix->mma_ready = false;   // the bf16 mirror and the norms are built lazily, as after an add
        }
    }
    if (st) {
        gorse_b200_vecdb_destroy(db);
        return st;
    }
    db->hidden.swap(hidden);
    db->dead.swap(dead);
    db->ts.swap(ts);
    db->cat_off.swap(cat_off);
    db->cats.swap(cats);
    db->live = n;
    db->meta_dirty = true;
    db->gen++;
    *out = db;
    if (bytes_out) *bytes_out = r.pos;
    return GORSE_B200_OK;
}

// ---- the neighbour cache's stream (gorse_b200_vecdb_neighbour_cache_save / _load) ----------------------------------------
//
// Slots are written as live ranks (a slot's position among the live slots, gorse_b200_vecdb_save's new_slot_out), so a stream
// saved from a collection with deleted slots loads into the collection its snapshot restores.  The header carries a
// fingerprint of everything the lists depend on, so a stream never loads into another collection.

constexpr char NBR_MAGIC[8] = {'G', 'B', '2', '0', '0', 'N', 'B', 'R'};
constexpr uint32_t NBR_VERSION = 1;
constexpr int NBR_THREADS = 256;
constexpr int64_t NBR_AHEAD_BYTES = 4ll << 20;   // load reads at most this far past the field it parses

struct NbrHeader {
    char magic[8];
    uint32_t version;
    int32_t n, dim, distance;
    int64_t live;
    uint64_t fingerprint;
    int64_t rows;
};
static_assert(sizeof(NbrHeader) == 48, "the neighbour stream header is 48 bytes without padding");

// The fingerprint's terms, one warp per live rank r (slot live_slot[r], hidden flag hidden[r]): the row's hash is the sum of
// mix64(index << 32 | fp32 bits) over its values (dense: every column, a bf16 value widened first; sparse: each (index,
// value) entry), and mix64(row hash + mix64(seed ^ (r << 1 | hidden))) is added into *out.  Every sum is modulo 2^64, so the
// result depends on neither the lanes' nor the warps' order.
template <typename T>
__global__ void __launch_bounds__(NBR_THREADS)
ncache_fingerprint_kernel(const T *X, int dim, const int64_t *sp_off, const uint32_t *sp_ind, const float *sp_val, const int64_t *live_slot,
                          const uint8_t *hidden, int64_t live, uint64_t seed, unsigned long long *out)
{
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * NBR_THREADS) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * NBR_THREADS + threadIdx.x) >> 5; r < live; r += nw) {
        const int64_t s = live_slot[r];
        uint64_t h = 0;
        if (dim > 0) {
            const T *x = X + s * dim;
            for (int j = lane; j < dim; j += 32) h += mix64((uint64_t)j << 32 | __float_as_uint(widen(x[j])));
        } else {
            for (int64_t t = sp_off[s] + lane; t < sp_off[s + 1]; t += 32) h += mix64((uint64_t)sp_ind[t] << 32 | __float_as_uint(sp_val[t]));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
        if (lane == 0) atomicAdd(out, (unsigned long long)mix64(h + mix64(seed ^ ((uint64_t)r << 1 | hidden[r]))));
    }
}

// One save chunk of m rows, one warp per row i: pool row prow[i] of the neighbour cache as the stream's 32-bit words at
// out + woff[i] - woff[0]: the row's live rank rank[i], its entry count, then each entry as (the live rank of its slot, score
// bits).  Every neighbour of a held row is a live slot of the generation the row belongs to.
__global__ void __launch_bounds__(NBR_THREADS)
ncache_gather_kernel(const uint2 *pool, const int32_t *pool_cnt, int n, const int32_t *prow, const int32_t *rank, const int64_t *woff, int64_t m,
                     const int32_t *rank_of_slot, uint32_t *out)
{
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * NBR_THREADS) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * NBR_THREADS + threadIdx.x) >> 5; i < m; i += nw) {
        const int32_t p = prow[i];
        const int c = pool_cnt[p];
        uint32_t *o = out + (woff[i] - woff[0]);
        if (lane == 0) {
            o[0] = (uint32_t)rank[i];
            o[1] = (uint32_t)c;
        }
        const uint2 *e = pool + (int64_t)p * n;
        for (int j = lane; j < c; j += 32) {
            const uint2 x = e[j];
            o[2 + 2 * j] = (uint32_t)rank_of_slot[x.x];
            o[3 + 2 * j] = x.y;
        }
    }
}

// the live slots of db in slot order (live_slot[rank]); rank_of_slot (may be nullptr): [slots], -1 for a deleted slot
void live_ranks(const gorse_b200_vecdb *db, std::vector<int64_t> &live_slot, std::vector<int32_t> *rank_of_slot)
{
    live_slot.clear();
    live_slot.reserve((size_t)db->live);
    if (rank_of_slot) rank_of_slot->assign(db->dead.size(), -1);
    for (size_t s = 0; s < db->dead.size(); s++) {
        if (db->dead[s]) continue;
        if (rank_of_slot) (*rank_of_slot)[s] = (int32_t)live_slot.size();
        live_slot.push_back((int64_t)s);
    }
}

// The fingerprint of what db's neighbour lists at n depend on: the kind, distance, dim, live count and n, then each live
// vector in rank order (its hidden flag and its values) through ncache_fingerprint_kernel.  The caller holds db->mu, the
// index's lock and the device.
int32_t ncache_fingerprint(gorse_b200_vecdb *db, int n, const std::vector<int64_t> &live_slot, uint64_t *fp)
{
    gorse_b200_ctx *c = db->ctx;
    const int64_t live = (int64_t)live_slot.size();
    uint64_t seed = mix64(NBR_VERSION);
    for (int64_t v : {(int64_t)(db->dim == 0), (int64_t)db->distance, (int64_t)db->dim, live, (int64_t)n}) seed = mix64(seed ^ (uint64_t)v);
    std::vector<uint8_t> hid((size_t)live);
    for (int64_t r = 0; r < live; r++) hid[(size_t)r] = db->hidden[(size_t)live_slot[(size_t)r]];
    DevBuf<int64_t> d_slot;
    DevBuf<uint8_t> d_hid;
    DevBuf<unsigned long long> d_sum;
    GB_TRY(d_slot.upload(live_slot.data(), (size_t)live, c->stream));
    GB_TRY(d_hid.upload(hid.data(), (size_t)live, c->stream));
    GB_TRY(d_sum.alloc(1));
    GB_CUDA(cudaMemsetAsync(d_sum.p, 0, sizeof(unsigned long long), c->stream));
    if (live > 0) {
        const unsigned grid = (unsigned)std::min<int64_t>(div_up(live * 32, NBR_THREADS), (int64_t)c->sm_count * 16);
        if (db->dim > 0) {
            with_rows(db->dense->rows(), [&](auto x) {
                ncache_fingerprint_kernel<<<grid, NBR_THREADS, 0, c->stream>>>(x, db->dim, nullptr, nullptr, nullptr, d_slot.p, d_hid.p, live, seed,
                                                                              d_sum.p);
            });
        } else {
            gorse_b200_sparse_index *sx = db->sparse;
            GB_TRY(sparse_sync_device(sx));
            ncache_fingerprint_kernel<float><<<grid, NBR_THREADS, 0, c->stream>>>(nullptr, 0, sx->off.p, sx->ind.p, sx->val.p, d_slot.p, d_hid.p,
                                                                                  live, seed, d_sum.p);
        }
        c->launches++;
        GB_CUDA(cudaGetLastError());
    }
    unsigned long long sum = 0;
    GB_CUDA(cudaMemcpyAsync(&sum, d_sum.p, sizeof(sum), cudaMemcpyDeviceToHost, c->stream));
    GB_CUDA(cudaStreamSynchronize(c->stream));
    *fp = mix64(seed ^ (uint64_t)sum);
    return GORSE_B200_OK;
}

int32_t ncache_off(const char *who)
{
    set_error("neighbour cache %s: the collection's neighbour cache is off", who);
    return GORSE_B200_ERR_STATE;
}

int32_t ncache_save(gorse_b200_vecdb *db, gorse_b200_write_fn write, void *user, int64_t *bytes_out)
{
    std::lock_guard<std::mutex> lk(db->mu);
    const NeighbourCache &K = db->ncache;
    if (K.cap == 0) return ncache_off("save");
    std::lock_guard<std::mutex> lk2(db->dense ? db->dense->mu : db->sparse->mu);
    gorse_b200_ctx *c = db->ctx;
    ScopedDevice sd(c->device);
    StreamSync sync{c->stream, c->copy_stream};
    const int n = K.n;
    std::vector<int64_t> live_slot;
    std::vector<int32_t> rank_of_slot;
    live_ranks(db, live_slot, &rank_of_slot);
    NbrHeader h{};
    memcpy(h.magic, NBR_MAGIC, sizeof(NBR_MAGIC));
    h.version = NBR_VERSION;
    h.n = n;
    h.dim = db->dim;
    h.distance = db->distance;
    h.live = (int64_t)live_slot.size();
    GB_TRY(ncache_fingerprint(db, n, live_slot, &h.fingerprint));
    // the held rows in ascending rank; a cache of an older generation holds nothing (it empties at its next read)
    std::vector<int32_t> prow, rank;
    if (K.gen == db->gen)
        for (int64_t r = 0; r < h.live; r++) {
            const int32_t p = K.row_of_slot[(size_t)live_slot[(size_t)r]];
            if (p < 0) continue;
            prow.push_back(p);
            rank.push_back((int32_t)r);
        }
    const int64_t rows = (int64_t)prow.size();
    h.rows = rows;
    std::vector<int32_t> cnt((size_t)K.used);
    if (rows > 0) {
        GB_CUDA(cudaMemcpyAsync(cnt.data(), K.cnt.p, sizeof(int32_t) * (size_t)K.used, cudaMemcpyDeviceToHost, c->stream));
        GB_CUDA(cudaStreamSynchronize(c->stream));
    }
    std::vector<int64_t> woff((size_t)rows + 1, 0);   // each row's first 32-bit word after the header
    for (int64_t i = 0; i < rows; i++) woff[(size_t)i + 1] = woff[(size_t)i] + 2 + 2 * (int64_t)cnt[(size_t)prow[(size_t)i]];
    Staging stg(c);
    const int64_t cap = std::min(STAGE_BYTES, std::max(MIN_STAGE_BYTES, 4 * woff[(size_t)rows]));   // a row is at most 8 + 8 * 1024 bytes
    GB_TRY(stg.alloc(cap, rows > 0 ? 2 : 1, rows > 0));
    Writer w{write, user, stg.h[0].p, cap, 0, 0, "neighbour cache save"};
    GB_TRY(w.put(&h, sizeof(h)));
    GB_TRY(w.flush());
    if (rows > 0) {
        // chunk k = rows [r0[k], r0[k + 1]) of at most cap bytes
        std::vector<int64_t> r0{0};
        while (r0.back() < rows) {
            int64_t e = r0.back();
            while (e < rows && 4 * (woff[(size_t)e + 1] - woff[(size_t)r0.back()]) <= cap) e++;
            r0.push_back(e);
        }
        const int64_t chunks = (int64_t)r0.size() - 1;
        DevBuf<int32_t> d_prow, d_rank, d_ros;
        DevBuf<int64_t> d_woff;
        GB_TRY(d_prow.upload(prow.data(), prow.size(), c->stream));
        GB_TRY(d_rank.upload(rank.data(), rank.size(), c->stream));
        GB_TRY(d_ros.upload(rank_of_slot.data(), rank_of_slot.size(), c->stream));
        GB_TRY(d_woff.upload(woff.data(), woff.size(), c->stream));
        auto bytes_of = [&](int64_t k) { return 4 * (woff[(size_t)r0[(size_t)k + 1]] - woff[(size_t)r0[(size_t)k]]); };
        GB_TRY(write_chunks(stg, w, chunks, bytes_of, [&](int64_t k, float *d) {
            const int64_t i0 = r0[(size_t)k], m = r0[(size_t)k + 1] - i0;
            const unsigned grid = (unsigned)std::min<int64_t>(div_up(m * 32, NBR_THREADS), (int64_t)c->sm_count * 16);
            ncache_gather_kernel<<<grid, NBR_THREADS, 0, c->stream>>>(K.entry.p, K.cnt.p, n, d_prow.p + i0, d_rank.p + i0, d_woff.p + i0, m, d_ros.p,
                                                                      reinterpret_cast<uint32_t *>(d));
        }));
    }
    if (bytes_out) *bytes_out = w.pos;
    return GORSE_B200_OK;
}

// the reader behind load's parser: take() hands out the next k bytes, reading ahead at most `more` bytes (capped at
// NBR_AHEAD_BYTES) that a well-formed stream holds after them, so the call never reads past the stream's end
struct Ahead {
    Reader &r;
    std::vector<char> buf;
    size_t at = 0, end = 0;
    int64_t pos() const { return r.pos - (int64_t)(end - at); }
    int32_t take(void *dst, int64_t k, int64_t more)
    {
        if ((int64_t)(end - at) < k) {
            memmove(buf.data(), buf.data() + at, end - at);
            end -= at;
            at = 0;
            const int64_t want = k - (int64_t)end + std::min(more, NBR_AHEAD_BYTES);
            buf.resize(end + (size_t)want);
            GB_TRY(r.get(buf.data() + end, want, "rows"));
            end += (size_t)want;
        }
        memcpy(dst, buf.data() + at, (size_t)k);
        at += (size_t)k;
        return GORSE_B200_OK;
    }
};

int32_t ncache_load(gorse_b200_vecdb *db, gorse_b200_read_fn read, void *user, int64_t *stats_out)
{
    std::lock_guard<std::mutex> lk(db->mu);
    NeighbourCache &K = db->ncache;
    if (K.cap == 0) return ncache_off("load");
    std::lock_guard<std::mutex> lk2(db->dense ? db->dense->mu : db->sparse->mu);
    gorse_b200_ctx *c = db->ctx;
    ScopedDevice sd(c->device);
    StreamSync sync{c->stream, c->copy_stream};
    Reader r{read, user, 0, "neighbour cache load"};
    NbrHeader h;
    GB_TRY(r.get(&h, sizeof(h), "header"));
    STREAM_CHECK(r, memcmp(h.magic, NBR_MAGIC, sizeof(NBR_MAGIC)) == 0, "magic", 0, "not a gorse_b200 neighbour cache stream");
    STREAM_CHECK(r, h.version == NBR_VERSION, "version", 8, "unknown version");
    if (h.n != K.n) {
        set_error("neighbour cache load: the stream holds lists of n = %d, the cache keeps n = %d", h.n, K.n);
        return GORSE_B200_ERR_STATE;
    }
    const int n = K.n;
    STREAM_CHECK(r, h.dim == db->dim, "dim", 16, "not the collection's");
    STREAM_CHECK(r, h.distance == db->distance, "distance", 20, "not the collection's");
    std::vector<int64_t> live_slot;
    live_ranks(db, live_slot, nullptr);
    const int64_t live = (int64_t)live_slot.size();
    STREAM_CHECK(r, h.live == live, "live count", 24, "not the collection's");
    uint64_t fp = 0;
    GB_TRY(ncache_fingerprint(db, n, live_slot, &fp));
    STREAM_CHECK(r, h.fingerprint == fp, "fingerprint", 32, "not the collection's: saved from another collection, or before a change of this one");
    STREAM_CHECK(r, h.rows >= 0 && h.rows <= live, "row count", 40, "negative or above the live count");
    // the rows the pool keeps (the lowest ranks) go into device staging in chunks of R rows through two pinned buffers (R n
    // entries, then R counts); the pool is touched only once the whole stream has been read and checked
    const int64_t rows = h.rows, kept = std::min(rows, K.cap);
    const int64_t R = std::max<int64_t>(1, std::min<int64_t>(kept, STAGE_BYTES / (8ll * n + 4)));
    DevBuf<uint2> s_entry;
    DevBuf<int32_t> s_cnt;
    Staging stg(c);
    if (kept > 0) {
        GB_TRY(s_entry.alloc((size_t)(kept * n)));
        GB_TRY(s_cnt.alloc((size_t)kept));
        GB_TRY(stg.alloc(R * (8ll * n + 4), 2, false));
    }
    std::vector<int64_t> kept_slot((size_t)kept);
    std::vector<uint2> spill((size_t)n);
    Ahead a{r};
    cudaError_t e = cudaSuccess;
    int64_t prev = -1;
    for (int64_t i = 0; i < rows; i++) {
        const int64_t at = a.pos(), k = i / R, j = i % R;
        const int b = (int)(k & 1);
        int32_t rc[2];
        GB_TRY(a.take(rc, 8, 8 * (rows - i - 1)));
        STREAM_CHECK(r, rc[0] >= 0 && rc[0] < live, "row rank", at, "outside [0, live count)");
        STREAM_CHECK(r, rc[0] > prev, "row rank", at, "not above the previous row's");
        STREAM_CHECK(r, rc[1] >= 0 && rc[1] <= n, "entry count", at + 4, "outside [0, n]");
        prev = rc[0];
        if (i < kept && j == 0) {
            e = stg.wait_free(k);
            if (e != cudaSuccess) break;
        }
        uint2 *row = i < kept ? reinterpret_cast<uint2 *>(stg.h[b].p) + j * n : spill.data();
        GB_TRY(a.take(row, 8ll * rc[1], 8 * (rows - i - 1)));
        for (int t = 0; t < rc[1]; t++) {
            STREAM_CHECK(r, (int32_t)row[t].x >= 0 && (int32_t)row[t].x < live, "entry rank", at + 8 + 8ll * t, "outside [0, live count)");
            row[t].x = (uint32_t)live_slot[row[t].x];
        }
        if (i >= kept) continue;
        kept_slot[(size_t)i] = live_slot[(size_t)rc[0]];
        int32_t *cnt = reinterpret_cast<int32_t *>(reinterpret_cast<uint2 *>(stg.h[b].p) + R * n);
        cnt[j] = rc[1];
        if (j == R - 1 || i == kept - 1) {
            const int64_t m = j + 1;
            e = cudaMemcpyAsync(s_entry.p + k * R * n, stg.h[b].p, sizeof(uint2) * (size_t)(m * n), cudaMemcpyHostToDevice, c->copy_stream);
            if (e == cudaSuccess) e = cudaMemcpyAsync(s_cnt.p + k * R, cnt, sizeof(int32_t) * (size_t)m, cudaMemcpyHostToDevice, c->copy_stream);
            if (e == cudaSuccess) e = stg.in_flight(k);
            if (e != cudaSuccess) break;
        }
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->copy_stream);
    if (e != cudaSuccess) {
        set_error("neighbour cache load: %s", cudaGetErrorString(e));
        return GORSE_B200_ERR_CUDA;
    }
    // every check has passed: the stream's rows replace the held ones, in pool rows 0 .. kept - 1
    ncache_reset(db);
    if (kept > 0) {
        e = cudaMemcpyAsync(K.entry.p, s_entry.p, sizeof(uint2) * (size_t)(kept * n), cudaMemcpyDeviceToDevice, c->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(K.cnt.p, s_cnt.p, sizeof(int32_t) * (size_t)kept, cudaMemcpyDeviceToDevice, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) {
            set_error("neighbour cache load: %s", cudaGetErrorString(e));
            return GORSE_B200_ERR_CUDA;
        }
    }
    for (int64_t i = 0; i < kept; i++) K.row_of_slot[(size_t)kept_slot[(size_t)i]] = (int32_t)i;
    K.used = kept;
    const int64_t st[3] = {kept, rows - kept, r.pos};
    if (stats_out) std::copy(st, st + 3, stats_out);
    return GORSE_B200_OK;
}

// one of the entries below: a host allocation that throws is GORSE_B200_ERR_OOM, naming the call
template <typename F>
int32_t guard(const char *who, F f)
{
    try {
        return f();
    } catch (const std::bad_alloc &) {
        set_error("%s: host allocation failed", who);
        return GORSE_B200_ERR_OOM;
    }
}

}  // namespace
}  // namespace gb

using namespace gb;

extern "C" {

int32_t gorse_b200_vecdb_save(gorse_b200_vecdb *db, gorse_b200_write_fn write, void *user, int64_t *new_slot_out, int64_t *bytes_out)
{
    GB_CHECK_ARG(db != nullptr && write != nullptr, "NULL collection or write callback");
    return guard("snapshot save", [&] { return save(db, write, user, new_slot_out, bytes_out); });
}

int32_t gorse_b200_vecdb_load(gorse_b200_ctx *ctx, gorse_b200_read_fn read, void *user, gorse_b200_vecdb **out, int64_t *bytes_out)
{
    GB_CHECK_ARG(ctx != nullptr && read != nullptr && out != nullptr, "NULL context, read callback or out");
    *out = nullptr;
    return guard("snapshot load", [&] { return load(ctx, read, user, out, bytes_out); });
}

int32_t gorse_b200_vecdb_neighbour_cache_save(gorse_b200_vecdb *db, gorse_b200_write_fn write, void *user, int64_t *bytes_out)
{
    GB_CHECK_ARG(db != nullptr && write != nullptr, "NULL collection or write callback");
    return guard("neighbour cache save", [&] { return ncache_save(db, write, user, bytes_out); });
}

int32_t gorse_b200_vecdb_neighbour_cache_load(gorse_b200_vecdb *db, gorse_b200_read_fn read, void *user, int64_t *stats_out)
{
    GB_CHECK_ARG(db != nullptr && read != nullptr, "NULL collection or read callback");
    return guard("neighbour cache load", [&] { return ncache_load(db, read, user, stats_out); });
}

}  // extern "C"
