/*
 * gorse_oracle.c -- CPU ORACLE (test infrastructure, never shipped, never on the product path).
 * See gorse_oracle.h for the parity status of each part.
 *
 * Build with -ffp-contract=off: every fused multiply-add below is an explicit fmaf() that
 * mirrors an FMA instruction in the reference's committed assembly
 * (common/floats/floats_avx512.s), everything else rounds once per operation like the
 * reference's Go code built with GOAMD64=v1.
 */
#define _GNU_SOURCE
#include "gorse_oracle.h"
#include <dlfcn.h>
#include <math.h>
#include <sched.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------------------------------
 * common/floats -- AVX-512 variants (what floats_amd64.go:39-53 dispatches on this host).
 * 16-lane body, 8-lane block, scalar tail; which of them fuse is read off the committed asm:
 *   body  : vfmadd (fused)                 floats_avx512.s:134,140
 *   8-lane: vmulps + vaddps (two roundings) floats_avx512.s:160-161
 *   tail  : vfmadd213ss (fused)            floats_avx512.s:181
 * ---------------------------------------------------------------------------------------- */

void gbo_mul_const_add_to(const float *a, float b, const float *c, float *dst, int64_t n)
{
    int64_t body = (n / 16) * 16, i = 0;
    for (; i < body; i++) dst[i] = fmaf(a[i], b, c[i]);
    if (n - i >= 8) {
        for (int k = 0; k < 8; k++, i++) { float m = a[i] * b; dst[i] = m + c[i]; }
    }
    for (; i < n; i++) dst[i] = fmaf(a[i], b, c[i]);
}

void gbo_mul_const_add(const float *a, float c, float *dst, int64_t n)
{
    int64_t body = (n / 16) * 16, i = 0;
    for (; i < body; i++) dst[i] = fmaf(a[i], c, dst[i]);
    if (n - i >= 8) {
        for (int k = 0; k < 8; k++, i++) { float m = a[i] * c; dst[i] = m + dst[i]; }
    }
    for (; i < n; i++) dst[i] = fmaf(a[i], c, dst[i]);
}

void gbo_mul_const_to(const float *a, float c, float *dst, int64_t n)
{
    for (int64_t i = 0; i < n; i++) dst[i] = a[i] * c;
}

void gbo_mul_const(float *a, float c, int64_t n)
{
    for (int64_t i = 0; i < n; i++) a[i] = a[i] * c;
}

void gbo_sub_to(const float *a, const float *b, float *c, int64_t n)
{
    for (int64_t i = 0; i < n; i++) c[i] = a[i] - b[i];
}

/* fixed reduce tree of the 16-lane accumulator: floats_avx512.c:327-339 */
static inline float tree16(const float *s)
{
    float r8[8], r4[4];
    for (int l = 0; l < 8; l++) r8[l] = s[l + 8] + s[l];
    for (int l = 0; l < 4; l++) r4[l] = r8[l + 4] + r8[l];
    float e = r4[0] + r4[2];
    float o = r4[1] + r4[3];
    return e + o;
}
/* 8-lane block tree: floats_avx512.c:349-358 */
static inline float tree8(const float *p)
{
    float q4[4];
    for (int l = 0; l < 4; l++) q4[l] = p[l + 4] + p[l];
    float e = q4[0] + q4[2];
    float o = q4[1] + q4[3];
    return e + o;
}

float gbo_dot(const float *a, const float *b, int64_t n)
{
    int64_t epoch = n / 16, remain = n % 16;
    float s[16];
    for (int l = 0; l < 16; l++) s[l] = 0.0f;
    if (epoch > 0)
        for (int l = 0; l < 16; l++) s[l] = a[l] * b[l];
    for (int64_t c = 1; c < epoch; c++)
        for (int l = 0; l < 16; l++) s[l] = fmaf(a[16 * c + l], b[16 * c + l], s[l]);
    float sum = tree16(s);
    a += 16 * epoch;
    b += 16 * epoch;
    if (remain >= 8) {
        float p[8];
        for (int l = 0; l < 8; l++) p[l] = a[l] * b[l];
        sum = sum + tree8(p);
        a += 8;
        b += 8;
        remain -= 8;
    }
    for (int64_t i = 0; i < remain; i++) sum = fmaf(a[i], b[i], sum);
    return sum;
}

float gbo_euclidean(const float *a, const float *b, int64_t n)
{
    int64_t epoch = n / 16, remain = n % 16;
    float s[16];
    for (int l = 0; l < 16; l++) s[l] = 0.0f;
    if (epoch > 0)
        for (int l = 0; l < 16; l++) { float v = a[l] - b[l]; s[l] = v * v; }
    for (int64_t c = 1; c < epoch; c++)
        for (int l = 0; l < 16; l++) { float v = a[16 * c + l] - b[16 * c + l]; v = v * v; s[l] = v + s[l]; }
    float sum = tree16(s);
    a += 16 * epoch;
    b += 16 * epoch;
    if (remain >= 8) {
        float p[8];
        for (int l = 0; l < 8; l++) { float v = a[l] - b[l]; p[l] = v * v; }
        sum = sum + tree8(p);
        a += 8;
        b += 8;
        remain -= 8;
    }
    for (int64_t i = 0; i < remain; i++) { float v = a[i] - b[i]; sum = fmaf(v, v, sum); }
    return sqrtf(sum);
}

/* common/floats/floats.go:21-33 (the generic Go loops; what a machine without AVX runs) */
float gbo_dot_scalar(const float *a, const float *b, int64_t n)
{
    float r = 0;
    for (int64_t i = 0; i < n; i++) { float m = a[i] * b[i]; r = r + m; }
    return r;
}
float gbo_euclidean_scalar(const float *a, const float *b, int64_t n)
{
    float r = 0;
    for (int64_t i = 0; i < n; i++) { float v = a[i] - b[i]; float m = v * v; r = r + m; }
    return sqrtf(r);
}

/* ------------------------------------------------------------------------------------------
 * chewxy/math32 v1.11.1 (go.mod:13), not in the reference.  PARITY UNPINNED.
 * Exp: the FreeBSD e_expf.c algorithm (argument reduction x = k*ln2 + r with a split float32 ln2,
 * degree-5 minimax on r*r, Ldexp) in the form of math32's portable exp.go.  Used at
 * model/cf/model.go:470-471.  Every operation rounds to float32 individually.
 * ---------------------------------------------------------------------------------------- */
float gbo_exp(float x)
{
    /* e_expf.c constants as carried by math32's exp.go */
    const float Ln2Hi = 6.9313812256e-01f; /* 0x3f317180 */
    const float Ln2Lo = 9.0580006145e-06f; /* 0x3717f7d1 */
    const float Log2e = 1.4426950216e+00f;
    const float Overflow = 7.09782712893383973096e+02f;
    const float Underflow = -7.45133219101941108420e+02f;
    const float NearZero = 1.0f / (float)(1 << 28);
    const float P1 = 1.6666667163e-01f;  /* 0x3e2aaaab */
    const float P2 = -2.7777778450e-03f; /* 0xbb360b61 */
    const float P3 = 6.6137559770e-05f;  /* 0x388ab355 */
    const float P4 = -1.6533901999e-06f; /* 0xb5ddea0e */
    const float P5 = 4.1381369442e-08f;  /* 0x3331bb4c */
    if (isnan(x) || (isinf(x) && x > 0)) return x;
    if (isinf(x) && x < 0) return 0.0f;
    if (x > Overflow) return INFINITY;
    if (x < Underflow) return 0.0f;
    if (-NearZero < x && x < NearZero) return 1.0f + x;
    int k = 0;
    if (x < 0) { float t = Log2e * x; t = t - 0.5f; k = (int)t; }
    else if (x > 0) { float t = Log2e * x; t = t + 0.5f; k = (int)t; }
    float kf = (float)k;
    float hi = kf * Ln2Hi; hi = x - hi;
    float lo = kf * Ln2Lo;
    float r = hi - lo;
    float t = r * r;
    float c = t * P5; c = P4 + c; c = t * c; c = P3 + c; c = t * c; c = P2 + c; c = t * c; c = P1 + c; c = t * c;
    c = r - c;
    float num = r * c;
    float den = 2.0f - c;
    float y = num / den;
    y = lo - y;
    y = y - hi;
    y = 1.0f - y;
    return ldexpf(y, k);
}

/* math32.Log2: frexp, Log(frac)*(1/Ln2) + exp.  Used at model/cf/evaluator.go:79,85.
 * Pinned only through the NDCG known answer (1e-5). */
float gbo_log2(float x)
{
    int e;
    float frac = frexpf(x, &e);
    if (frac == 0.5f) return (float)(e - 1);
    float l = logf(frac);
    float inv = (float)(1.0 / 0.693147180559945309417232121458176568);
    l = l * inv;
    return l + (float)e;
}

/* ------------------------------------------------------------------------------------------
 * Go container/heap restated from its documented algorithm (SURVEY Appendix B) with
 * heap._heap.Less = strict weight compare (common/heap/pq.go:42-48).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    gbo_elem *e;
    int64_t n, cap;
    int desc;
} goheap;

static void gh_init(goheap *h, int desc, int64_t cap)
{
    h->e = (gbo_elem *)malloc(sizeof(gbo_elem) * (size_t)(cap > 4 ? cap : 4));
    h->n = 0;
    h->cap = cap > 4 ? cap : 4;
    h->desc = desc;
}
static void gh_free(goheap *h) { free(h->e); h->e = NULL; }
static inline int gh_less(const goheap *h, int64_t i, int64_t j)
{
    return h->desc ? (h->e[i].weight > h->e[j].weight) : (h->e[i].weight < h->e[j].weight);
}
static inline void gh_swap(goheap *h, int64_t i, int64_t j)
{
    gbo_elem t = h->e[i]; h->e[i] = h->e[j]; h->e[j] = t;
}
static void gh_up(goheap *h, int64_t j)
{
    for (;;) {
        int64_t i = (j - 1) / 2; /* Go integer division truncates toward zero */
        if (i == j || !gh_less(h, j, i)) break;
        gh_swap(h, i, j);
        j = i;
    }
}
static void gh_down(goheap *h, int64_t i0, int64_t n)
{
    int64_t i = i0;
    for (;;) {
        int64_t j1 = 2 * i + 1;
        if (j1 >= n || j1 < 0) break;
        int64_t j = j1, j2 = j1 + 1;
        if (j2 < n && gh_less(h, j2, j1)) j = j2;
        if (!gh_less(h, j, i)) break;
        gh_swap(h, i, j);
        i = j;
    }
}
static void gh_push(goheap *h, int32_t v, float w)
{
    if (h->n == h->cap) {
        h->cap *= 2;
        h->e = (gbo_elem *)realloc(h->e, sizeof(gbo_elem) * (size_t)h->cap);
    }
    h->e[h->n].value = v;
    h->e[h->n].weight = w;
    h->n++;
    gh_up(h, h->n - 1);
}
static gbo_elem gh_pop(goheap *h)
{
    int64_t n = h->n - 1;
    gh_swap(h, 0, n);
    gh_down(h, 0, n);
    gbo_elem it = h->e[h->n - 1];
    h->n--;
    return it;
}

/* TopKFilter: common/heap/filter.go:35-59 (min-heap, desc=false) */
int32_t gbo_topk_filter(const int32_t *values, const float *weights, int64_t n, int32_t k,
                        int32_t *out_values, float *out_weights)
{
    goheap h;
    gh_init(&h, 0, (int64_t)k + 2);
    for (int64_t t = 0; t < n; t++) {
        gh_push(&h, values[t], weights[t]);
        if (h.n > k) (void)gh_pop(&h);
    }
    int32_t m = (int32_t)h.n;
    for (int32_t i = m - 1; i >= 0; i--) {
        gbo_elem e = gh_pop(&h);
        out_values[i] = e.value;
        if (out_weights) out_weights[i] = e.weight;
    }
    gh_free(&h);
    return m;
}

/* PriorityQueue with its never-shrinking lookup set: common/heap/pq.go:69-131 */
typedef struct {
    goheap h;
    int32_t *set; /* open addressing, -1 empty */
    int64_t set_cap, set_n;
} gopq;
static void pq_set_init(gopq *p, int64_t cap)
{
    int64_t c = 16;
    while (c < cap * 2) c *= 2;
    p->set = (int32_t *)malloc(sizeof(int32_t) * (size_t)c);
    for (int64_t i = 0; i < c; i++) p->set[i] = -1;
    p->set_cap = c;
    p->set_n = 0;
}
static int pq_set_contains_or_add(gopq *p, int32_t v, int add)
{
    if (add && (p->set_n + 1) * 2 > p->set_cap) {
        int32_t *old = p->set;
        int64_t oc = p->set_cap;
        pq_set_init(p, oc);
        for (int64_t i = 0; i < oc; i++)
            if (old[i] >= 0) pq_set_contains_or_add(p, old[i], 1);
        free(old);
    }
    uint64_t hsh = (uint64_t)(uint32_t)v * 0x9E3779B97F4A7C15ull;
    int64_t m = p->set_cap - 1, pos = (int64_t)(hsh >> 20) & m;
    while (p->set[pos] >= 0) {
        if (p->set[pos] == v) return 1;
        pos = (pos + 1) & m;
    }
    if (add) { p->set[pos] = v; p->set_n++; }
    return 0;
}
static void pq_init(gopq *p, int desc, int64_t cap)
{
    gh_init(&p->h, desc, cap);
    pq_set_init(p, cap);
}
static void pq_free(gopq *p) { gh_free(&p->h); free(p->set); }
static void pq_push(gopq *p, int32_t v, float w)
{
    if (isnan(w)) abort(); /* pq.go:82-83 panics */
    if (!pq_set_contains_or_add(p, v, 0)) {
        gh_push(&p->h, v, w);
        pq_set_contains_or_add(p, v, 1);
    }
}
static void pq_reverse(const gopq *p, gopq *out)
{
    pq_init(out, !p->h.desc, p->h.n + 1);
    for (int64_t i = 0; i < p->h.n; i++) pq_push(out, p->h.e[i].value, p->h.e[i].weight);
}

int32_t gbo_pq_push_pop_all(const int32_t *values, const float *weights, int64_t n, int32_t desc,
                            int32_t reverse_first, int32_t *out_values, float *out_weights)
{
    gopq p;
    pq_init(&p, desc, n + 1);
    for (int64_t i = 0; i < n; i++) pq_push(&p, values[i], weights[i]);
    gopq *use = &p, r;
    if (reverse_first) { pq_reverse(&p, &r); use = &r; }
    int32_t m = 0;
    while (use->h.n > 0) {
        gbo_elem e = gh_pop(&use->h);
        out_values[m] = e.value;
        out_weights[m] = e.weight;
        m++;
    }
    if (reverse_first) pq_free(&r);
    pq_free(&p);
    return m;
}

/* ------------------------------------------------------------------------------------------
 * BPR: model/cf/model.go:469-488 (SURVEY Appendix A for the rounding sequence).
 * Optional binding to the reference's own kernels (oracle/_ref) for cross-validation and for
 * the CPU baseline.
 * ---------------------------------------------------------------------------------------- */
typedef float (*ref_dot_fn)(float *, float *, int64_t);
typedef void (*ref_mct_fn)(float *, float *, float *, int64_t);
typedef void (*ref_mc_fn)(float *, float *, int64_t);
static struct {
    void *handle;
    ref_dot_fn dot, euclidean;
    ref_mct_fn mul_const_to, mul_const_add, sub_to;
    ref_mc_fn mul_const;
} g_ref;

int32_t gbo_ref_bind(const char *path)
{
    void *h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
    if (!h) return -1;
    g_ref.dot = (ref_dot_fn)dlsym(h, "_mm512_dot");
    g_ref.euclidean = (ref_dot_fn)dlsym(h, "_mm512_euclidean");
    g_ref.mul_const_to = (ref_mct_fn)dlsym(h, "_mm512_mul_const_to");
    g_ref.mul_const_add = (ref_mct_fn)dlsym(h, "_mm512_mul_const_add");
    g_ref.sub_to = (ref_mct_fn)dlsym(h, "_mm512_sub_to");
    g_ref.mul_const = (ref_mc_fn)dlsym(h, "_mm512_mul_const");
    if (!g_ref.dot || !g_ref.euclidean || !g_ref.mul_const_to || !g_ref.mul_const_add || !g_ref.sub_to ||
        !g_ref.mul_const) {
        dlclose(h);
        memset(&g_ref, 0, sizeof(g_ref));
        return -2;
    }
    g_ref.handle = h;
    return 0;
}

#define GBO_MAX_D 4096

void gbo_bpr_step(float *P, float *Q, int32_t d, int32_t u, int32_t i, int32_t j, float lr, float reg)
{
    float *Pu = P + (int64_t)u * d, *Qi = Q + (int64_t)i * d, *Qj = Q + (int64_t)j * d;
    float temp[GBO_MAX_D], uf[GBO_MAX_D], pf[GBO_MAX_D], nf[GBO_MAX_D];
    /* :469 */
    float diff = gbo_dot(Pu, Qi, d) - gbo_dot(Pu, Qj, d);
    /* :471 (the :470 cost accumulation is dead code) */
    float e = gbo_exp(-diff);
    float grad = e / (1.0f + e);
    /* :473-475 */
    memcpy(uf, Pu, sizeof(float) * (size_t)d);
    memcpy(pf, Qi, sizeof(float) * (size_t)d);
    memcpy(nf, Qj, sizeof(float) * (size_t)d);
    /* :477-479 */
    gbo_mul_const_to(uf, grad, temp, d);
    gbo_mul_const_add(pf, -reg, temp, d);
    gbo_mul_const_add(temp, lr, Qi, d);
    /* :481-483 */
    gbo_mul_const_to(uf, -grad, temp, d);
    gbo_mul_const_add(nf, -reg, temp, d);
    gbo_mul_const_add(temp, lr, Qj, d);
    /* :485-488 */
    gbo_sub_to(pf, nf, temp, d);
    gbo_mul_const(temp, grad, d);
    gbo_mul_const_add(uf, -reg, temp, d);
    gbo_mul_const_add(temp, lr, Pu, d);
}

void gbo_bpr_apply_triples(float *P, float *Q, int32_t d, const int32_t *uij, int64_t n, float lr, float reg)
{
    for (int64_t t = 0; t < n; t++) {
        if (uij[3 * t + 2] < 0) continue; /* sampler's "no valid negative" marker */
        gbo_bpr_step(P, Q, d, uij[3 * t], uij[3 * t + 1], uij[3 * t + 2], lr, reg);
    }
}

/* same step through the reference's own compiled kernels (only when oracle/_ref is bound) */
static void bpr_step_ref(float *P, float *Q, int32_t d, int32_t u, int32_t i, int32_t j, float lr, float reg,
                         float *temp, float *uf, float *pf, float *nf)
{
    float *Pu = P + (int64_t)u * d, *Qi = Q + (int64_t)i * d, *Qj = Q + (int64_t)j * d;
    float diff = g_ref.dot(Pu, Qi, d) - g_ref.dot(Pu, Qj, d);
    float e = gbo_exp(-diff);
    float grad = e / (1.0f + e), ngrad = -grad, nreg = -reg;
    memcpy(uf, Pu, sizeof(float) * (size_t)d);
    memcpy(pf, Qi, sizeof(float) * (size_t)d);
    memcpy(nf, Qj, sizeof(float) * (size_t)d);
    g_ref.mul_const_to(uf, &grad, temp, d);
    g_ref.mul_const_add(pf, &nreg, temp, d);
    g_ref.mul_const_add(temp, &lr, Qi, d);
    g_ref.mul_const_to(uf, &ngrad, temp, d);
    g_ref.mul_const_add(nf, &nreg, temp, d);
    g_ref.mul_const_add(temp, &lr, Qj, d);
    g_ref.sub_to(pf, nf, temp, d);
    g_ref.mul_const(temp, &grad, d);
    g_ref.mul_const_add(uf, &nreg, temp, d);
    g_ref.mul_const_add(temp, &lr, Pu, d);
}

/* ---- counter-based sampler (ours; DESIGN.md "sampling").  Distribution = model.go:449-468:
 * u uniform over users with >=1 feedback, i uniform in R_u, j uniform over items rejected while in R_u. */
static inline uint64_t mix64(uint64_t z)
{
    z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27; z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}
typedef struct { uint64_t x; } sstream;
static inline uint32_t s_next32(sstream *s)
{
    s->x += 0x9E3779B97F4A7C15ull;
    return (uint32_t)(mix64(s->x) >> 32);
}
static inline uint32_t s_bounded(sstream *s, uint32_t n)
{
    uint64_t m = (uint64_t)s_next32(s) * n;
    uint32_t l = (uint32_t)m;
    if (l < n) {
        uint32_t t = (0u - n) % n;
        while (l < t) { m = (uint64_t)s_next32(s) * n; l = (uint32_t)m; }
    }
    return (uint32_t)(m >> 32);
}
static inline int row_contains(const int32_t *row, int64_t len, int32_t v)
{
    int64_t lo = 0, hi = len;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (row[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo < len && row[lo] == v;
}
static inline void sample_one(int32_t n_items, const int64_t *user_off, const int32_t *user_items,
                              const int32_t *active, int32_t n_active, uint64_t base, int64_t step,
                              int32_t *out)
{
    sstream s;
    s.x = mix64(base + (uint64_t)step);
    int32_t u = active[s_bounded(&s, (uint32_t)n_active)];
    int64_t o = user_off[u], len = user_off[u + 1] - o;
    int32_t i = user_items[o + s_bounded(&s, (uint32_t)len)];
    int32_t j = -1;
    if (len < n_items) {
        for (;;) {
            int32_t c = (int32_t)s_bounded(&s, (uint32_t)n_items);
            if (!row_contains(user_items + o, len, c)) { j = c; break; }
        }
    }
    out[0] = u; out[1] = i; out[2] = j;
}

void gbo_bpr_sample_triples(int32_t n_items, const int64_t *user_off, const int32_t *user_items,
                            const int32_t *active_users, int32_t n_active,
                            uint64_t seed, int64_t first_step, int64_t n, int32_t *uij_out)
{
    uint64_t base = mix64(seed);
    for (int64_t t = 0; t < n; t++)
        sample_one(n_items, user_off, user_items, active_users, n_active, base, first_step + t, uij_out + 3 * t);
}

/* ---- dataset.SampleUserNegatives (dataset/dataset.go:242-253) -> util.SampleInt32 (common/util/random.go:108-132).
 * Per user: the union of train(u) and test(u) is excluded; when n_cand >= n_items - |excluded| every remaining item is
 * returned ascending (:116-122), else items are drawn uniformly and rejected while excluded or already drawn (:124-130).
 * Go's math/rand stream cannot be reproduced (SURVEY F9): the draws come from the counter RNG shared with the CUDA
 * path (stream = mix64(seed ^ C) + global user id).  train rows must be sorted ascending (the device copy is).
 * Two calls: neg_items_out == NULL fills neg_off_out only. */
void gbo_sample_user_negatives(int32_t n_items, int32_t n_users, int32_t u_base, const int64_t *train_off, const int32_t *train_items,
                               const int64_t *test_off, const int32_t *test_items, int32_t n_cand, uint64_t seed,
                               int64_t *neg_off_out, int32_t *neg_items_out)
{
    const uint64_t base = mix64(seed ^ 0xbb67ae8584caa73bull);
    neg_off_out[0] = 0;
    for (int32_t u = 0; u < n_users; u++) {
        const int32_t *tr = train_items + train_off[u], *te = test_items + test_off[u];
        const int64_t ntr = train_off[u + 1] - train_off[u], nte = test_off[u + 1] - test_off[u];
        int64_t card = 0;
        for (int64_t a = 0; a < ntr; a++) if (a == 0 || tr[a] != tr[a - 1]) card++;
        for (int64_t a = 0; a < nte; a++) {
            int dup = row_contains(tr, ntr, te[a]);
            for (int64_t b = 0; b < a && !dup; b++) dup = te[b] == te[a];
            if (!dup) card++;
        }
        const int64_t n = (int64_t)n_cand >= (int64_t)n_items - card ? (int64_t)n_items - card : (int64_t)n_cand;
        neg_off_out[u + 1] = neg_off_out[u] + n;
        if (!neg_items_out) continue;
        int32_t *out = neg_items_out + neg_off_out[u];
        int64_t k = 0;
        if (n < n_cand) {
            for (int32_t v = 0; v < n_items && k < n; v++) {
                int ex = row_contains(tr, ntr, v);
                for (int64_t a = 0; a < nte && !ex; a++) ex = te[a] == v;
                if (!ex) out[k++] = v;
            }
            continue;
        }
        sstream s;
        s.x = mix64(base + (uint64_t)(u_base + u));
        while (k < n) {
            const int32_t v = (int32_t)s_bounded(&s, (uint32_t)n_items);
            int ex = row_contains(tr, ntr, v);
            for (int64_t a = 0; a < nte && !ex; a++) ex = te[a] == v;
            for (int64_t b = 0; b < k && !ex; b++) ex = out[b] == v;
            if (!ex) out[k++] = v;
        }
    }
}

/* ---- CPU-arm reproducibility (VERDICT r1: the Hogwild baseline moved 6 -> 27 M triples/s between runs): worker t is
 * pinned to the t-th CPU of the process's affinity mask, and the factor tables can be first-touched page-interleaved
 * over the workers so that the random row accesses spread over all NUMA nodes instead of the allocating thread's. */
static cpu_set_t g_aff;
static int g_aff_n = -1;
static void aff_init(void)
{
    if (g_aff_n >= 0) return;
    CPU_ZERO(&g_aff);
    g_aff_n = sched_getaffinity(0, sizeof(g_aff), &g_aff) == 0 ? CPU_COUNT(&g_aff) : 0;
}
static void pin_self(int t)
{
    if (g_aff_n <= 0) return;
    int want = t % g_aff_n, seen = 0;
    for (int c = 0; c < CPU_SETSIZE; c++) {
        if (!CPU_ISSET(c, &g_aff)) continue;
        if (seen++ == want) {
            cpu_set_t one;
            CPU_ZERO(&one);
            CPU_SET(c, &one);
            pthread_setaffinity_np(pthread_self(), sizeof(one), &one);
            return;
        }
    }
}
typedef struct { float *buf; int64_t n; float std; uint64_t base; int t, nt; } fill_job;
static void *fill_worker(void *arg)
{
    fill_job *jb = (fill_job *)arg;
    pin_self(jb->t);
    const int64_t page = 1024;   /* floats per 4 KB page */
    for (int64_t p0 = (int64_t)jb->t * page; p0 < jb->n; p0 += (int64_t)jb->nt * page) {
        const int64_t p1 = p0 + page < jb->n ? p0 + page : jb->n;
        for (int64_t i = p0; i < p1; i += 2) {
            /* Box-Muller on the counter RNG: a pair of N(0, std) per counter */
            uint64_t z = mix64(jb->base + (uint64_t)i);
            float u1 = ((float)(uint32_t)(z >> 40) + 0.5f) * (1.0f / 16777216.0f);
            float u2 = ((float)(uint32_t)((z >> 8) & 0xffffff) + 0.5f) * (1.0f / 16777216.0f);
            float r = sqrtf(-2.0f * logf(u1)) * jb->std;
            jb->buf[i] = r * cosf(6.2831853f * u2);
            if (i + 1 < p1) jb->buf[i + 1] = r * sinf(6.2831853f * u2);
        }
    }
    return NULL;
}
void gbo_fill_normal_interleaved(float *buf, int64_t n, float std, uint64_t seed, int32_t n_threads)
{
    aff_init();
    if (n_threads < 1) n_threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)n_threads);
    fill_job *jobs = (fill_job *)malloc(sizeof(fill_job) * (size_t)n_threads);
    for (int t = 0; t < n_threads; t++) {
        fill_job jb = {buf, n, std, mix64(seed ^ 0x3c6ef372fe94f82bull), t, n_threads};
        jobs[t] = jb;
        pthread_create(&th[t], NULL, fill_worker, &jobs[t]);
    }
    for (int t = 0; t < n_threads; t++) pthread_join(th[t], NULL);
    free(th);
    free(jobs);
}

static double now_sec(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

typedef struct {
    float *P, *Q;
    int32_t n_items, d;
    const int64_t *user_off;
    const int32_t *user_items, *active;
    int32_t n_active;
    uint64_t base;
    int64_t s0, s1;
    float lr, reg;
    int use_ref, tid;
} bpr_job;

static void *bpr_worker(void *arg)
{
    bpr_job *jb = (bpr_job *)arg;
    pin_self(jb->tid);
    float *scratch = (float *)malloc(sizeof(float) * 4 * (size_t)jb->d);
    for (int64_t s = jb->s0; s < jb->s1; s++) {
        int32_t t[3];
        sample_one(jb->n_items, jb->user_off, jb->user_items, jb->active, jb->n_active, jb->base, s, t);
        if (t[2] < 0) continue;
        if (jb->use_ref)
            bpr_step_ref(jb->P, jb->Q, jb->d, t[0], t[1], t[2], jb->lr, jb->reg, scratch, scratch + jb->d,
                         scratch + 2 * jb->d, scratch + 3 * jb->d);
        else
            gbo_bpr_step(jb->P, jb->Q, jb->d, t[0], t[1], t[2], jb->lr, jb->reg);
    }
    free(scratch);
    return NULL;
}

/* Hogwild over n_threads (model.go:448 with Jobs=n_threads, minus Go's channel/mutex costs):
 * the CPU baseline.  Lock-free, non-atomic, like the reference. */
double gbo_bpr_epoch_threads(float *P, float *Q, int32_t n_items, int32_t d,
                             const int64_t *user_off, const int32_t *user_items,
                             const int32_t *active_users, int32_t n_active,
                             uint64_t seed, int64_t n_steps, float lr, float reg, int32_t n_threads,
                             int32_t use_ref_kernels)
{
    if (n_threads < 1) n_threads = 1;
    if (use_ref_kernels && !g_ref.handle) use_ref_kernels = 0;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)n_threads);
    bpr_job *jobs = (bpr_job *)malloc(sizeof(bpr_job) * (size_t)n_threads);
    uint64_t base = mix64(seed);
    aff_init();
    double t0 = now_sec();
    for (int t = 0; t < n_threads; t++) {
        bpr_job jb = {P, Q, n_items, d, user_off, user_items, active_users, n_active, base,
                      n_steps * t / n_threads, n_steps * (t + 1) / n_threads, lr, reg, use_ref_kernels, t};
        jobs[t] = jb;
        pthread_create(&th[t], NULL, bpr_worker, &jobs[t]);
    }
    for (int t = 0; t < n_threads; t++) pthread_join(th[t], NULL);
    double t1 = now_sec();
    free(th);
    free(jobs);
    return t1 - t0;
}

/* ------------------------------------------------------------------------------------------
 * ALS / eALS ("CCD"): model/cf/model.go:641-738.  Scalar Go loops, every op rounds to fp32.
 * ---------------------------------------------------------------------------------------- */
static void als_gram(const float *X, int32_t rows, int32_t d, const int64_t *off, float *s)
{
    /* :645-658 / :693-706 -- rows in index order, skipping rows without feedback */
    memset(s, 0, sizeof(float) * (size_t)d * (size_t)d);
    for (int32_t r = 0; r < rows; r++) {
        if (off[r + 1] - off[r] > 0) {
            const float *x = X + (int64_t)r * d;
            for (int i = 0; i < d; i++)
                for (int j = 0; j < d; j++) { float m = x[i] * x[j]; s[i * d + j] = s[i * d + j] + m; }
        }
    }
}

/* one row update, :660-685 (users) / :708-733 (items): X = table being updated, Y = the other one */
static void als_row(float *xrow, const float *Y, int32_t d, const int32_t *fb, int64_t n, const float *s,
                    float reg, float w, float *pred, float *res)
{
    for (int64_t t = 0; t < n; t++) pred[t] = gbo_dot(xrow, Y + (int64_t)fb[t] * d, d); /* internalPredict */
    float omw = 1.0f - w;
    for (int f = 0; f < d; f++) {
        for (int64_t t = 0; t < n; t++) {
            float m = xrow[f] * Y[(int64_t)fb[t] * d + f];
            res[t] = pred[t] - m;
        }
        float a = 0, b = 0, c = 0;
        for (int64_t t = 0; t < n; t++) {
            float y = Y[(int64_t)fb[t] * d + f];
            float t1 = omw * res[t]; t1 = 1.0f - t1; t1 = t1 * y; a = a + t1;
            float t2 = omw * y; t2 = t2 * y; c = c + t2;
        }
        for (int k = 0; k < d; k++)
            if (k != f) { float t3 = w * xrow[k]; t3 = t3 * s[k * d + f]; b = b + t3; }
        float num = a - b;
        float den = w * s[f * d + f]; den = c + den; den = den + reg;
        xrow[f] = num / den;
        for (int64_t t = 0; t < n; t++) {
            float m = xrow[f] * Y[(int64_t)fb[t] * d + f];
            pred[t] = res[t] + m;
        }
    }
}

void gbo_als_epoch(float *P, float *Q, int32_t n_users, int32_t n_items, int32_t d,
                   const int64_t *user_off, const int32_t *user_items,
                   const int64_t *item_off, const int32_t *item_users, float reg, float alpha)
{
    float *s = (float *)malloc(sizeof(float) * (size_t)d * (size_t)d);
    int64_t maxlen = 1;
    for (int32_t u = 0; u < n_users; u++) if (user_off[u + 1] - user_off[u] > maxlen) maxlen = user_off[u + 1] - user_off[u];
    for (int32_t i = 0; i < n_items; i++) if (item_off[i + 1] - item_off[i] > maxlen) maxlen = item_off[i + 1] - item_off[i];
    float *pred = (float *)malloc(sizeof(float) * (size_t)maxlen);
    float *res = (float *)malloc(sizeof(float) * (size_t)maxlen);
    als_gram(Q, n_items, d, item_off, s);
    for (int32_t u = 0; u < n_users; u++)
        als_row(P + (int64_t)u * d, Q, d, user_items + user_off[u], user_off[u + 1] - user_off[u], s, reg, alpha, pred, res);
    als_gram(P, n_users, d, user_off, s);
    for (int32_t i = 0; i < n_items; i++)
        als_row(Q + (int64_t)i * d, P, d, item_users + item_off[i], item_off[i + 1] - item_off[i], s, reg, alpha, pred, res);
    free(s); free(pred); free(res);
}

typedef struct {
    float *X; const float *Y; int32_t d; const int64_t *off; const int32_t *fb; const float *s;
    float reg, w; int32_t r0, r1; int64_t maxlen;
} als_job;
static void *als_worker(void *arg)
{
    als_job *jb = (als_job *)arg;
    float *pred = (float *)malloc(sizeof(float) * (size_t)jb->maxlen * 2);
    for (int32_t r = jb->r0; r < jb->r1; r++)
        als_row(jb->X + (int64_t)r * jb->d, jb->Y, jb->d, jb->fb + jb->off[r], jb->off[r + 1] - jb->off[r], jb->s,
                jb->reg, jb->w, pred, pred + jb->maxlen);
    free(pred);
    return NULL;
}
static void als_half_threads(float *X, const float *Y, int32_t rows, int32_t d, const int64_t *off, const int32_t *fb,
                             const float *s, float reg, float w, int nt, int64_t maxlen)
{
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nt);
    als_job *jobs = (als_job *)malloc(sizeof(als_job) * (size_t)nt);
    for (int t = 0; t < nt; t++) {
        als_job jb = {X, Y, d, off, fb, s, reg, w, (int32_t)((int64_t)rows * t / nt), (int32_t)((int64_t)rows * (t + 1) / nt), maxlen};
        jobs[t] = jb;
        pthread_create(&th[t], NULL, als_worker, &jobs[t]);
    }
    for (int t = 0; t < nt; t++) pthread_join(th[t], NULL);
    free(th); free(jobs);
}
/* CPU baseline: rows in parallel (model.go:659,707 with Jobs=n_threads), Gram serial as in the reference */
double gbo_als_epoch_threads(float *P, float *Q, int32_t n_users, int32_t n_items, int32_t d,
                   const int64_t *user_off, const int32_t *user_items,
                   const int64_t *item_off, const int32_t *item_users, float reg, float alpha,
                   int32_t n_threads)
{
    if (n_threads < 1) n_threads = 1;
    float *s = (float *)malloc(sizeof(float) * (size_t)d * (size_t)d);
    int64_t maxlen = 1;
    for (int32_t u = 0; u < n_users; u++) if (user_off[u + 1] - user_off[u] > maxlen) maxlen = user_off[u + 1] - user_off[u];
    for (int32_t i = 0; i < n_items; i++) if (item_off[i + 1] - item_off[i] > maxlen) maxlen = item_off[i + 1] - item_off[i];
    double t0 = now_sec();
    als_gram(Q, n_items, d, item_off, s);
    als_half_threads(P, Q, n_users, d, user_off, user_items, s, reg, alpha, n_threads, maxlen);
    als_gram(P, n_users, d, user_off, s);
    als_half_threads(Q, P, n_items, d, item_off, item_users, s, reg, alpha, n_threads, maxlen);
    double t1 = now_sec();
    free(s);
    return t1 - t0;
}

/* ------------------------------------------------------------------------------------------
 * Bruteforce: common/ann/bruteforce.go:39-83
 * ---------------------------------------------------------------------------------------- */
static inline float metric_dist(const float *a, const float *b, int32_t d, int32_t metric)
{
    if (metric == GBO_METRIC_EUCLIDEAN) return gbo_euclidean(a, b, d);
    return -gbo_dot(a, b, d); /* logics/cf.go:32-34 */
}

int32_t gbo_bruteforce_search(const float *X, int64_t N, int32_t d, const float *q, int64_t self,
                              int32_t k, int32_t prune0, int32_t metric,
                              int32_t *out_idx, float *out_score)
{
    gopq pq;
    pq_init(&pq, 1, (int64_t)k + 2);
    /* the lookup set only ever sees distinct ids here; size it lazily */
    for (int64_t i = 0; i < N; i++) {
        if (i == self) continue; /* :47 */
        pq_push(&pq, (int32_t)i, metric_dist(q, X + i * d, d, metric));
        if (pq.h.n > k) (void)gh_pop(&pq.h);
    }
    gopq r;
    pq_reverse(&pq, &r);
    int32_t m = 0;
    while (r.h.n > 0) {
        gbo_elem e = gh_pop(&r.h);
        if (!prune0 || e.weight > 0) { out_idx[m] = e.value; out_score[m] = e.weight; m++; }
    }
    pq_free(&r);
    pq_free(&pq);
    return m;
}

typedef struct {
    const float *X; int64_t N; int32_t d; int64_t q0, q1, qbase; int32_t k, prune0, metric;
    int32_t *out_idx; float *out_score; int32_t *out_count;
} bf_job;
static void *bf_worker(void *arg)
{
    bf_job *jb = (bf_job *)arg;
    for (int64_t q = jb->q0; q < jb->q1; q++) {
        int64_t row = q - jb->qbase;
        int32_t *oi = jb->out_idx + row * jb->k;
        float *os = jb->out_score + row * jb->k;
        int32_t m = gbo_bruteforce_search(jb->X, jb->N, jb->d, jb->X + q * jb->d, q, jb->k, jb->prune0, jb->metric, oi, os);
        for (int32_t t = m; t < jb->k; t++) { oi[t] = -1; os[t] = 0; }
        if (jb->out_count) jb->out_count[row] = m;
    }
    return NULL;
}
double gbo_bruteforce_all(const float *X, int64_t N, int32_t d, int64_t q0, int64_t q1, int32_t k,
                          int32_t prune0, int32_t metric, int32_t n_threads,
                          int32_t *out_idx, float *out_score, int32_t *out_count)
{
    if (n_threads < 1) n_threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)n_threads);
    bf_job *jobs = (bf_job *)malloc(sizeof(bf_job) * (size_t)n_threads);
    double t0 = now_sec();
    int64_t nq = q1 - q0;
    for (int t = 0; t < n_threads; t++) {
        bf_job jb = {X, N, d, q0 + nq * t / n_threads, q0 + nq * (t + 1) / n_threads, q0, k, prune0, metric, out_idx, out_score, out_count};
        jobs[t] = jb;
        pthread_create(&th[t], NULL, bf_worker, &jobs[t]);
    }
    for (int t = 0; t < n_threads; t++) pthread_join(th[t], NULL);
    double t1 = now_sec();
    free(th); free(jobs);
    return t1 - t0;
}

/* Test helper, not a reference function: sum over observed (u,i) of (1 - r)^2 - w r^2 with r = p_u . q_i, the data
 * part of the objective one eALS epoch (model.go:641-738) cannot increase; accumulated in double, rows over threads.
 * tests/als_checks.py adds the Gram and regularisation terms. */
typedef struct { const float *P, *Q; int32_t d; const int64_t *off; const int32_t *items; double w; int32_t u0, u1; double out; } obj_job;
static void *obj_worker(void *arg)
{
    obj_job *jb = (obj_job *)arg;
    double acc = 0.0;
    for (int32_t u = jb->u0; u < jb->u1; u++) {
        const float *p = jb->P + (int64_t)u * jb->d;
        for (int64_t t = jb->off[u]; t < jb->off[u + 1]; t++) {
            const float *q = jb->Q + (int64_t)jb->items[t] * jb->d;
            double r = 0.0;
            for (int32_t k = 0; k < jb->d; k++) r += (double)p[k] * (double)q[k];
            acc += (1.0 - r) * (1.0 - r) - jb->w * r * r;
        }
    }
    jb->out = acc;
    return NULL;
}
double gbo_als_observed_loss(const float *P, const float *Q, int32_t n_users, int32_t d, const int64_t *user_off,
                             const int32_t *user_items, double w, int32_t n_threads)
{
    if (n_threads < 1) n_threads = 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)n_threads);
    obj_job *jobs = (obj_job *)malloc(sizeof(obj_job) * (size_t)n_threads);
    for (int t = 0; t < n_threads; t++) {
        obj_job jb = {P, Q, d, user_off, user_items, w, (int32_t)((int64_t)n_users * t / n_threads),
                      (int32_t)((int64_t)n_users * (t + 1) / n_threads), 0.0};
        jobs[t] = jb;
        pthread_create(&th[t], NULL, obj_worker, &jobs[t]);
    }
    double tot = 0.0;
    for (int t = 0; t < n_threads; t++) { pthread_join(th[t], NULL); tot += jobs[t].out; }
    free(th); free(jobs);
    return tot;
}

/* ------------------------------------------------------------------------------------------
 * Similarity vectors and scores: logics/item_to_item.go, logics/user_to_user.go, logics/vector_writer.go
 * ---------------------------------------------------------------------------------------- */
/* dense embedding as stored: bfloats.FromFloat32 keeps the high 16 bits (common/bfloats/bfloats.go:23-29),
 * bfloats.ToFloat32 widens them again (:31-37); logics/item_to_item.go:151-164 ExtractItemEmbedding */
void gbo_bf16_truncate(const float *in, int64_t n, float *out)
{
    for (int64_t i = 0; i < n; i++) {
        uint32_t u;
        memcpy(&u, &in[i], 4);
        u = (uint32_t)((uint16_t)(u >> 16)) << 16;
        memcpy(&out[i], &u, 4);
    }
}

/* appendSparseVector (logics/vector_writer.go:200-209): ids outside [0, len(idf)) or with idf <= 0 are skipped;
 * value = float32(math.Sqrt(float64(idf[id]))); "auto" calls it twice, the second time with offset = len(tagsIDF)
 * (logics/item_to_item.go:238-239).  Returns the number of entries appended. */
int32_t gbo_sparse_vector(const int32_t *ids, int32_t n_ids, const float *idf, int32_t n_idf, uint32_t offset,
                          uint32_t *indices_out, float *values_out)
{
    int32_t m = 0;
    for (int32_t t = 0; t < n_ids; t++) {
        int32_t id = ids[t];
        if (id < 0 || id >= n_idf || idf[id] <= 0) continue;
        indices_out[m] = offset + (uint32_t)id;
        values_out[m] = (float)sqrt((double)idf[id]);
        m++;
    }
    return m;
}

/* QueryItemToItem / QueryUserToUser post-processing (logics/item_to_item.go:63-85, user_to_user.go:63-85).
 * Input: the neighbours as the vector store returned them for a query of n+1, score = "higher is closer"
 * (Dot: the dot product; Euclidean: the NEGATED distance, storage/vectors/database.go:101).  Drops the query's own
 * id, drops score <= 0 for Dot, scales, maps Euclidean to 1/(1 - score) = 1/(1 + dist), stops at n. */
int32_t gbo_similar_scores(int32_t euclidean, double score_scale, int32_t self_id, int32_t n,
                           const int32_t *nbr_ids, const float *nbr_score, int32_t n_nbr,
                           int32_t *ids_out, double *scores_out)
{
    int32_t m = 0;
    for (int32_t t = 0; t < n_nbr && m < n; t++) {
        if (nbr_ids[t] == self_id || (!euclidean && nbr_score[t] <= 0)) continue;
        double score = (double)nbr_score[t] * score_scale;
        if (euclidean) score = 1 / (1 - score);
        ids_out[m] = nbr_ids[t];
        scores_out[m] = score;
        m++;
    }
    return m;
}

/* Sparse similarity search (the "tags" / "users" / "auto" item-to-item and user-to-user types): what the reference
 * asks its vector store for with sparse vectors and the Dot metric (storage/vectors/xvec.go:244-248 flat sparse index,
 * :405 query).  The arithmetic lives in gorse-io/xvec v0.0.0-20260821023012-cf0c34c6025f (go.mod:31), which is NOT under
 * the reference: PARITY UNPINNED except for the neighbour-id orders the reference's tests assert
 * (logics/item_to_item_test.go:212-316).  Restated as: indices ascending in every vector (item_to_item.go:191,213,
 * 236-237 sort the ids before appendSparseVector), dot = merge-join summed in index order in fp32, the k largest dots
 * through the same bounded Go heap as Bruteforce (distance = -dot, ties as container/heap leaves them). */
float gbo_sparse_dot(const uint32_t *ia, const float *va, int32_t na, const uint32_t *ib, const float *vb, int32_t nb)
{
    float s = 0.0f;
    int32_t a = 0, b = 0;
    while (a < na && b < nb) {
        if (ia[a] == ib[b]) { s = s + va[a] * vb[b]; a++; b++; }
        else if (ia[a] < ib[b]) a++;
        else b++;
    }
    return s;
}

/* neighbours of stored vector `self` (or of nothing stored when self < 0 and q_* given): ids and dots, best first */
int32_t gbo_sparse_bruteforce_search(const int64_t *off, const uint32_t *indices, const float *values, int64_t N,
                                     const uint32_t *q_ind, const float *q_val, int32_t q_n, int64_t self, int32_t k,
                                     int32_t *out_idx, float *out_dot)
{
    gopq pq;
    pq_init(&pq, 1, (int64_t)k + 2);
    for (int64_t i = 0; i < N; i++) {
        if (i == self) continue;
        float dotv = gbo_sparse_dot(q_ind, q_val, q_n, indices + off[i], values + off[i], (int32_t)(off[i + 1] - off[i]));
        pq_push(&pq, (int32_t)i, -dotv);
        if (pq.h.n > k) (void)gh_pop(&pq.h);
    }
    gopq r;
    pq_reverse(&pq, &r);
    int32_t m = 0;
    while (r.h.n > 0) {
        gbo_elem e = gh_pop(&r.h);
        out_idx[m] = e.value; out_dot[m] = -e.weight; m++;
    }
    pq_free(&r);
    pq_free(&pq);
    return m;
}

/* ------------------------------------------------------------------------------------------
 * Metrics + Evaluate: model/cf/evaluator.go
 * ---------------------------------------------------------------------------------------- */
static inline int in_set(const int32_t *t, int32_t n, int32_t v)
{
    for (int32_t i = 0; i < n; i++) if (t[i] == v) return 1;
    return 0;
}
/* mapset cardinality: number of distinct ids */
static int32_t cardinality(const int32_t *t, int32_t n)
{
    int32_t c = 0;
    for (int32_t i = 0; i < n; i++) {
        int dup = 0;
        for (int32_t j = 0; j < i; j++) if (t[j] == t[i]) { dup = 1; break; }
        if (!dup) c++;
    }
    return c;
}
float gbo_ndcg(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank)
{
    int32_t card = cardinality(target, n_target);
    float idcg = 0;
    for (int32_t i = 0; i < card && i < n_rank; i++) { float l = gbo_log2((float)i + 2.0f); idcg = idcg + 1.0f / l; }
    float dcg = 0;
    for (int32_t i = 0; i < n_rank; i++)
        if (in_set(target, n_target, rank[i])) { float l = gbo_log2((float)i + 2.0f); dcg = dcg + 1.0f / l; }
    return dcg / idcg;
}
float gbo_precision(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank)
{
    float hit = 0;
    for (int32_t i = 0; i < n_rank; i++) if (in_set(target, n_target, rank[i])) hit = hit + 1.0f;
    return hit / (float)n_rank;
}
float gbo_recall(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank)
{
    int hit = 0;
    for (int32_t i = 0; i < n_rank; i++) if (in_set(target, n_target, rank[i])) hit++;
    return (float)hit / (float)cardinality(target, n_target);
}
float gbo_hr(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank)
{
    for (int32_t i = 0; i < n_rank; i++) if (in_set(target, n_target, rank[i])) return 1;
    return 0;
}
float gbo_map(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank)
{
    float sum = 0; int hit = 0;
    for (int32_t i = 0; i < n_rank; i++)
        if (in_set(target, n_target, rank[i])) { hit++; sum = sum + (float)hit / (float)(i + 1); }
    return sum / (float)cardinality(target, n_target);
}
float gbo_mrr(const int32_t *target, int32_t n_target, const int32_t *rank, int32_t n_rank)
{
    for (int32_t i = 0; i < n_rank; i++) if (in_set(target, n_target, rank[i])) return 1.0f / (float)(i + 1);
    return 0;
}

void gbo_evaluate(const float *P, const float *Q, int32_t n_users, int32_t d,
                  const int64_t *test_off, const int32_t *test_items,
                  const int64_t *neg_off, const int32_t *neg_items, int32_t topk, float out[3])
{
    float sum[3] = {0, 0, 0}, count = 0;
    int64_t maxc = 1;
    for (int32_t u = 0; u < n_users; u++) {
        int64_t c = (test_off[u + 1] - test_off[u]) + (neg_off[u + 1] - neg_off[u]);
        if (c > maxc) maxc = c;
    }
    int32_t *cand = (int32_t *)malloc(sizeof(int32_t) * (size_t)maxc);
    float *score = (float *)malloc(sizeof(float) * (size_t)maxc);
    int32_t *rank = (int32_t *)malloc(sizeof(int32_t) * (size_t)(topk > 0 ? topk : 1));
    for (int32_t u = 0; u < n_users; u++) {
        int32_t nt = (int32_t)(test_off[u + 1] - test_off[u]);
        if (nt <= 0) continue; /* :47 */
        int32_t nn = (int32_t)(neg_off[u + 1] - neg_off[u]);
        const int32_t *tgt = test_items + test_off[u];
        /* :51-53 candidates = test positives ++ negatives */
        memcpy(cand, tgt, sizeof(int32_t) * (size_t)nt);
        memcpy(cand + nt, neg_items + neg_off[u], sizeof(int32_t) * (size_t)nn);
        for (int32_t c = 0; c < nt + nn; c++) score[c] = gbo_dot(P + (int64_t)u * d, Q + (int64_t)cand[c] * d, d);
        int32_t nr = gbo_topk_filter(cand, score, nt + nn, topk, rank, NULL); /* Rank :162-169 */
        count = count + 1.0f;
        sum[0] = sum[0] + gbo_ndcg(tgt, nt, rank, nr);
        sum[1] = sum[1] + gbo_precision(tgt, nt, rank, nr);
        sum[2] = sum[2] + gbo_recall(tgt, nt, rank, nr);
    }
    float inv = 1.0f / count; /* :70-71 */
    gbo_mul_const(sum, inv, 3);
    out[0] = sum[0]; out[1] = sum[1]; out[2] = sum[2];
    free(cand); free(score); free(rank);
}
