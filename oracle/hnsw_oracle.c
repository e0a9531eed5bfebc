/* TEST INFRASTRUCTURE ONLY -- see hnsw_oracle.h.
 *
 * Plain-C restatement of the reference HNSW hot path.  "U/" = /root/reference/lantern_hnsw/
 * third_party/usearch/.  This file restates behaviour; it shares no code with the reference
 * (different data layout: SoA arrays + u32 ids instead of byte tapes + uint48 slots).
 * Parity status: pinned against oracle/_ref (the compiled reference) and the reference's golden
 * vectors by tests/test_oracle_ref.py and tests/test_golden.py.
 */
#define _GNU_SOURCE
#include "hnsw_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------
 * Scalar codecs.  U/include/usearch/index_plugins.hpp:879-974 (cast_gt family),
 * :310-329 (f16 via fp16 library = IEEE round-to-nearest-even), :934-964 (i8_converted_t).
 * ---------------------------------------------------------------------------------------- */
static uint32_t f32_bits(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
}
static float bits_f32(uint32_t u) {
    float f;
    memcpy(&f, &u, 4);
    return f;
}

float ora_f16_to_f32(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1Fu;
    uint32_t man = h & 0x3FFu;
    if (exp == 0) {
        if (man == 0)
            return bits_f32(sign);
        /* subnormal: value = man * 2^-24 */
        float v = (float)man * (1.0f / 16777216.0f);
        return sign ? -v : v;
    }
    if (exp == 31)
        return bits_f32(sign | 0x7F800000u | (man << 13));
    return bits_f32(sign | ((exp + 112u) << 23) | (man << 13));
}

uint16_t ora_f32_to_f16(float f) {
    uint32_t x = f32_bits(f);
    uint32_t sign = (x >> 16) & 0x8000u;
    uint32_t ax = x & 0x7FFFFFFFu;
    if (ax > 0x7F800000u)
        return (uint16_t)(sign | 0x7E00u); /* NaN */
    if (ax >= 0x47800000u)                 /* >= 65536 -> inf (65520 rounds to inf below) */
        return (uint16_t)(sign | 0x7C00u);
    if (ax < 0x33000000u) /* < 2^-25 -> 0 (exactly 2^-25 ties to even = 0) */
        return (uint16_t)sign;
    int32_t e = (int32_t)(ax >> 23) - 127;
    uint32_t m = (ax & 0x7FFFFFu) | 0x800000u;
    uint32_t shift, half;
    uint32_t out;
    if (e < -14) { /* subnormal half */
        shift = (uint32_t)(13 + (-14 - e));
        out = m >> shift;
        half = 1u << (shift - 1);
        uint32_t rem = m & ((1u << shift) - 1u);
        if (rem > half || (rem == half && (out & 1u)))
            out++;
        return (uint16_t)(sign | out);
    }
    out = ((uint32_t)(e + 15) << 10) | ((m >> 13) & 0x3FFu);
    uint32_t rem = m & 0x1FFFu;
    if (rem > 0x1000u || (rem == 0x1000u && (out & 1u)))
        out++; /* may carry into exponent, up to inf: correct */
    return (uint16_t)(sign | out);
}

static int8_t f32_to_i8(float v) { /* index_plugins.hpp:960-961: clamp(v*100, -100, 100) then truncation */
    float s = v * 100.0f;
    if (s < -100.0f)
        s = -100.0f;
    if (s > 100.0f)
        s = 100.0f;
    return (int8_t)s;
}

static size_t bytes_per_vector(int kind, size_t dims) {
    switch (kind) {
    case ORA_F32: return dims * 4;
    case ORA_F64: return dims * 8;
    case ORA_F16: return dims * 2;
    case ORA_I8: return dims;
    case ORA_B1: return (dims + 7) / 8;
    default: return 0;
    }
}

void ora_cast_f32(const float* in, size_t dims, int to_kind, void* out) {
    size_t i;
    switch (to_kind) {
    case ORA_F32: memcpy(out, in, dims * 4); break;
    case ORA_F16:
        for (i = 0; i < dims; ++i)
            ((uint16_t*)out)[i] = ora_f32_to_f16(in[i]);
        break;
    case ORA_I8:
        for (i = 0; i < dims; ++i)
            ((int8_t*)out)[i] = f32_to_i8(in[i]);
        break;
    case ORA_B1: /* index_plugins.hpp:909-918: bit i -> 128 >> (i & 7), set when x > 0 */
        memset(out, 0, (dims + 7) / 8);
        for (i = 0; i < dims; ++i)
            if (in[i] > 0)
                ((uint8_t*)out)[i / 8] |= (uint8_t)(128u >> (i & 7));
        break;
    default: break;
    }
}

/* ------------------------------------------------------------------------------------------
 * Metrics.  index_plugins.hpp:1004-1028 (cos), :1034-1051 (l2sq), :1058-1081 (hamming over
 * bytes), dispatch :1446-1522 (b1 storage forces hamming for cos/l2sq, :1465,:1477).
 * fp32 accumulation, sequential order (the reference's order is compiler-chosen; the parity
 * contract is 1e-5 relative).
 * ---------------------------------------------------------------------------------------- */
static float load_scalar(const void* p, int kind, size_t i) {
    switch (kind) {
    case ORA_F32: return ((const float*)p)[i];
    case ORA_F16: return ora_f16_to_f32(((const uint16_t*)p)[i]);
    case ORA_I8: return (float)((const int8_t*)p)[i];
    default: return 0.f;
    }
}

float ora_distance(const void* a, const void* b, int kind, size_t dims, int metric) {
    size_t i;
    if (kind == ORA_B1 || metric == ORA_METRIC_HAMMING) {
        size_t words = (dims + 7) / 8, matches = 0;
        const uint8_t *pa = (const uint8_t*)a, *pb = (const uint8_t*)b;
        for (i = 0; i < words; ++i)
            matches += (size_t)__builtin_popcount((unsigned)(pa[i] ^ pb[i]));
        return (float)matches;
    }
    if (kind == ORA_F64) {
        const double *pa = (const double*)a, *pb = (const double*)b;
        double ab = 0, a2 = 0, b2 = 0, l2 = 0;
        for (i = 0; i < dims; ++i) {
            ab += pa[i] * pb[i], a2 += pa[i] * pa[i], b2 += pb[i] * pb[i];
            l2 += (pa[i] - pb[i]) * (pa[i] - pb[i]);
        }
        if (metric == ORA_METRIC_L2SQ)
            return (float)l2;
        if (metric == ORA_METRIC_IP)
            return (float)(1 - ab);
        if (a2 == 0 && b2 == 0)
            return 0.f;
        if (a2 == 0 || b2 == 0)
            return 1.f;
        return (float)(1 - ab / (sqrt(a2) * sqrt(b2)));
    }
    if (metric == ORA_METRIC_L2SQ) {
        float acc = 0.f;
        for (i = 0; i < dims; ++i) {
            float d = load_scalar(a, kind, i) - load_scalar(b, kind, i);
            acc += d * d;
        }
        return acc;
    }
    {
        float ab = 0.f, a2 = 0.f, b2 = 0.f;
        for (i = 0; i < dims; ++i) {
            float x = load_scalar(a, kind, i), y = load_scalar(b, kind, i);
            ab += x * y, a2 += x * x, b2 += y * y;
        }
        if (metric == ORA_METRIC_IP)
            return 1.f - ab;
        /* cos: zero-norm table, index_plugins.hpp:1022-1026 */
        if (a2 == 0.f && b2 == 0.f)
            return 0.f;
        if (a2 == 0.f || b2 == 0.f)
            return 1.f;
        return 1.f - ab / (sqrtf(a2) * sqrtf(b2));
    }
}

/* ------------------------------------------------------------------------------------------
 * PQ codec.  U/include/usearch/lantern_storage.hpp:100-149.  Codebook tape float[centroid][dims];
 * subvector s of centroid c at c*dims + s*subdim.  Encode = per-subvector argmin, strict '<'
 * (lowest id wins).  compat128: the reference loop counter is a signed char (`byte_t c`,
 * :123) so centroids >= 128 are never visited.
 * ---------------------------------------------------------------------------------------- */
void ora_pq_compress(const float* codebook, size_t dims, size_t num_centroids, size_t num_subvectors,
                     const float* vector, uint8_t* codes, int compat128) {
    size_t subdim = dims / num_subvectors, s, c, i;
    size_t limit = (compat128 && num_centroids > 128) ? 128 : num_centroids;
    for (s = 0; s < num_subvectors; ++s) {
        float best = 3.402823466e+38f;
        uint8_t best_c = 0;
        for (c = 0; c < limit; ++c) {
            const float* cen = codebook + c * dims + s * subdim;
            float dist = 0.f;
            for (i = 0; i < subdim; ++i) {
                float d = vector[s * subdim + i] - cen[i];
                dist += d * d;
            }
            if (dist < best)
                best = dist, best_c = (uint8_t)c;
        }
        codes[s] = best_c;
    }
}

void ora_pq_decompress(const float* codebook, size_t dims, size_t num_centroids, size_t num_subvectors,
                       const uint8_t* codes, float* vector) {
    size_t subdim = dims / num_subvectors, s;
    (void)num_centroids;
    for (s = 0; s < num_subvectors; ++s)
        memcpy(vector + s * subdim, codebook + (size_t)codes[s] * dims + s * subdim, subdim * sizeof(float));
}

/* ------------------------------------------------------------------------------------------
 * Containers.  index.hpp:2062-2066 candidate_t (ordering by distance only);
 * :529-658 max_heap_gt (shift_up :637-640, shift_down :642-657, pop :615-622);
 * :668-780 sorted_buffer_gt (insert :752-763 = lower_bound, new goes BEFORE equal elements,
 * last evicted when full, rejected when slot == limit).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    float d;
    uint32_t s;
} cand_t;

typedef struct {
    cand_t* e;
    size_t n, cap;
} cvec_t;

static int cvec_reserve(cvec_t* v, size_t want) {
    if (want <= v->cap)
        return 1;
    size_t nc = v->cap ? v->cap : 16;
    while (nc < want)
        nc *= 2;
    cand_t* ne = (cand_t*)realloc(v->e, nc * sizeof(cand_t));
    if (!ne)
        return 0;
    v->e = ne, v->cap = nc;
    return 1;
}

static void heap_shift_up(cvec_t* h, size_t i) {
    while (i) {
        size_t p = (i - 1) / 2;
        if (!(h->e[p].d < h->e[i].d))
            break;
        cand_t t = h->e[p];
        h->e[p] = h->e[i], h->e[i] = t;
        i = p;
    }
}
static void heap_shift_down(cvec_t* h, size_t i) {
    for (;;) {
        size_t mx = i, l = 2 * i + 1, r = 2 * i + 2;
        if (l < h->n && h->e[mx].d < h->e[l].d)
            mx = l;
        if (r < h->n && h->e[mx].d < h->e[r].d)
            mx = r;
        if (mx == i)
            return;
        cand_t t = h->e[i];
        h->e[i] = h->e[mx], h->e[mx] = t;
        i = mx;
    }
}
static void heap_push(cvec_t* h, float d, uint32_t s) {
    cvec_reserve(h, h->n + 1);
    h->e[h->n].d = d, h->e[h->n].s = s;
    h->n++;
    heap_shift_up(h, h->n - 1);
}
static cand_t heap_pop(cvec_t* h) {
    cand_t top = h->e[0];
    h->e[0] = h->e[h->n - 1], h->e[h->n - 1] = top;
    h->n--;
    heap_shift_down(h, 0);
    return top;
}

static size_t sbuf_lower_bound(const cvec_t* b, float d) {
    size_t lo = 0, hi = b->n;
    while (lo < hi) {
        size_t mid = lo + (hi - lo) / 2;
        if (b->e[mid].d < d)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo;
}
static void sbuf_insert_reserved(cvec_t* b, float d, uint32_t s) { /* index.hpp:739-747 */
    cvec_reserve(b, b->n + 1);
    size_t slot = sbuf_lower_bound(b, d);
    memmove(b->e + slot + 1, b->e + slot, (b->n - slot) * sizeof(cand_t));
    b->e[slot].d = d, b->e[slot].s = s;
    b->n++;
}
static int sbuf_insert(cvec_t* b, float d, uint32_t s, size_t limit) { /* index.hpp:752-763 */
    size_t slot = sbuf_lower_bound(b, d);
    if (slot == limit)
        return 0;
    cvec_reserve(b, b->n + 1);
    size_t full = (b->n == limit);
    memmove(b->e + slot + 1, b->e + slot, (b->n - slot - full) * sizeof(cand_t));
    b->e[slot].d = d, b->e[slot].s = s;
    b->n += !full;
    return 1;
}

/* ------------------------------------------------------------------------------------------
 * Index.
 * ---------------------------------------------------------------------------------------- */
struct ora_index {
    int metric, quant, pq, compat128;
    size_t dims, M, M0, efc, ef;
    size_t ncent, nsub;
    const float* codebook; /* borrowed, like usearch_init (U/c/usearch.h:136-140) */
    size_t vec_bytes;      /* bytes of one vector in the metric's scalar kind */
    size_t stored_bytes;   /* what is kept per node: vec_bytes, or nsub codes when pq */
    size_t n, cap;
    uint64_t* keys;
    int16_t* levels;
    uint32_t* cnt0;
    uint32_t* nbr0;   /* [cap][M0] */
    uint32_t** upper; /* per node: level x (1 + M) u32 */
    uint8_t* vectors; /* [cap][stored_bytes] */
    int max_level;
    uint64_t entry;
    /* per-"thread" context (index.hpp:2078-2106): one context, single-threaded oracle */
    cvec_t next, top;
    uint32_t* visit;
    uint32_t epoch;
    uint32_t rng; /* std::default_random_engine == minstd_rand0, default seed 1 */
    int engine_order; /* 0 = the reference's heap; 1 = the CUDA engine's tie order (search and insertion beams) */
    float *dec_a, *dec_b;
    uint8_t* cast_buf;
    ora_stats st;
};

ora_index* ora_init(int metric, int quant, size_t dims, size_t connectivity, size_t expansion_add,
                    size_t expansion_search, int pq, size_t num_centroids, size_t num_subvectors,
                    const float* codebook, int pq_compat128) {
    if (pq && (num_centroids == 0 || num_subvectors == 0 || !codebook || num_centroids > 256 ||
               dims % num_subvectors != 0 || dims >= 2000))
        return NULL; /* U/c/lib.cpp:135-140, lantern_storage.hpp:90-94 */
    ora_index* x = (ora_index*)calloc(1, sizeof(ora_index));
    if (!x)
        return NULL;
    x->metric = metric, x->quant = quant, x->dims = dims;
    x->M = connectivity ? connectivity : 16; /* index.hpp:1249-1250 */
    x->M0 = x->M * 2;
    x->efc = expansion_add ? expansion_add : 128;
    x->ef = expansion_search ? expansion_search : 64;
    x->pq = pq, x->ncent = num_centroids, x->nsub = num_subvectors, x->codebook = codebook;
    x->compat128 = pq_compat128;
    x->vec_bytes = bytes_per_vector(quant, dims);
    x->stored_bytes = pq ? num_subvectors : x->vec_bytes;
    x->rng = 1u;
    x->max_level = -1;
    x->dec_a = (float*)malloc(dims * sizeof(float) + 16);
    x->dec_b = (float*)malloc(dims * sizeof(float) + 16);
    x->cast_buf = (uint8_t*)malloc(x->vec_bytes + 16);
    return x;
}

void ora_free(ora_index* x) {
    size_t i;
    if (!x)
        return;
    for (i = 0; i < x->n; ++i)
        free(x->upper ? x->upper[i] : NULL);
    free(x->keys), free(x->levels), free(x->cnt0), free(x->nbr0), free(x->upper), free(x->vectors);
    free(x->next.e), free(x->top.e), free(x->visit), free(x->dec_a), free(x->dec_b), free(x->cast_buf);
    free(x);
}

int ora_reserve(ora_index* x, size_t cap) {
    if (cap <= x->cap)
        return 1;
#define GROW(field, type, per)                                                                                         \
    do {                                                                                                               \
        type* p = (type*)realloc(x->field, cap * (per) * sizeof(type));                                                \
        if (!p)                                                                                                        \
            return 0;                                                                                                  \
        memset(p + x->cap * (per), 0, (cap - x->cap) * (per) * sizeof(type));                                          \
        x->field = p;                                                                                                  \
    } while (0)
    GROW(keys, uint64_t, 1);
    GROW(levels, int16_t, 1);
    GROW(cnt0, uint32_t, 1);
    GROW(nbr0, uint32_t, x->M0);
    GROW(upper, uint32_t*, 1);
    GROW(vectors, uint8_t, x->stored_bytes);
    GROW(visit, uint32_t, 1);
#undef GROW
    x->cap = cap;
    return 1;
}

size_t ora_size(const ora_index* x) { return x->n; }
void ora_set_engine_order(ora_index* x, int on) { x->engine_order = on; }
size_t ora_dimensions(const ora_index* x) { return x->dims; }
size_t ora_connectivity(const ora_index* x) { return x->M; }
int ora_max_level(const ora_index* x) { return x->max_level; }
uint64_t ora_entry_slot(const ora_index* x) { return x->entry; }
int ora_node_level(const ora_index* x, size_t slot) { return x->levels[slot]; }
uint64_t ora_node_key(const ora_index* x, size_t slot) { return x->keys[slot]; }
const void* ora_node_vector(const ora_index* x, size_t slot) { return x->vectors + slot * x->stored_bytes; }

static uint32_t* nbr_list(const ora_index* x, size_t slot, int level, uint32_t** count) {
    if (level == 0) {
        *count = &x->cnt0[slot];
        return x->nbr0 + slot * x->M0;
    }
    uint32_t* base = x->upper[slot] + (size_t)(level - 1) * (1 + x->M);
    *count = base;
    return base + 1;
}

size_t ora_node_neighbors(const ora_index* x, size_t slot, int level, uint32_t* out) {
    uint32_t* cnt;
    uint32_t* l = nbr_list(x, slot, level, &cnt);
    if (out)
        memcpy(out, l, *cnt * sizeof(uint32_t));
    return *cnt;
}

/* metric_proxy_t, U/include/usearch/index_dense.hpp:331-361: value-vs-member and member-vs-member;
 * with pq every stored operand is decompressed first (lantern_storage.hpp:264-267), the value
 * (query / new vector) never is.  Each call counts as one computed distance (index.hpp:2086-2104). */
static const void* stored_operand(ora_index* x, uint32_t slot, float* buf) {
    const uint8_t* p = x->vectors + (size_t)slot * x->stored_bytes;
    if (!x->pq)
        return p;
    ora_pq_decompress(x->codebook, x->dims, x->ncent, x->nsub, p, buf);
    return buf;
}
static float measure_qv(ora_index* x, const void* value, uint32_t slot) {
    x->st.computed_distances++;
    return ora_distance(value, stored_operand(x, slot, x->dec_b), x->quant, x->dims, x->metric);
}
static float measure_vv(ora_index* x, uint32_t a, uint32_t b) {
    x->st.computed_distances++;
    const void* pa = stored_operand(x, a, x->dec_a);
    const void* pb = stored_operand(x, b, x->dec_b);
    return ora_distance(pa, pb, x->quant, x->dims, x->metric);
}

static void visits_clear(ora_index* x) {
    if (++x->epoch == 0) {
        memset(x->visit, 0, x->cap * sizeof(uint32_t));
        x->epoch = 1;
    }
}
static int visits_set(ora_index* x, uint32_t s) { /* returns previous membership (index.hpp:995-1010) */
    int was = x->visit[s] == x->epoch;
    x->visit[s] = x->epoch;
    return was;
}

/* search_for_one_, index.hpp:3277-3316: greedy descent over levels (begin_level, end_level];
 * the neighbour list is that of the closest node at the START of a pass; strict '<'. */
static uint32_t search_for_one(ora_index* x, const void* q, uint32_t closest, int begin_level, int end_level) {
    float closest_d = measure_qv(x, q, closest);
    int level;
    for (level = begin_level; level > end_level; --level) {
        int changed;
        do {
            uint32_t* cnt;
            uint32_t* l = nbr_list(x, closest, level, &cnt);
            uint32_t n = *cnt, i;
            changed = 0;
            for (i = 0; i < n; ++i) {
                float d = measure_qv(x, q, l[i]);
                if (d < closest_d)
                    closest_d = d, closest = l[i], changed = 1;
            }
            x->st.visited_members++;
            x->st.upper_hops++;
        } while (changed);
    }
    return closest;
}

/* search_to_find_in_base_, index.hpp:3400-3485 (continue_search = false). */
static void search_base(ora_index* x, const void* q, uint32_t start, size_t top_limit) {
    cvec_t *next = &x->next, *top = &x->top;
    visits_clear(x);
    next->n = 0, top->n = 0;
    float radius = measure_qv(x, q, start);
    heap_push(next, -radius, start);
    sbuf_insert_reserved(top, radius, start);
    visits_set(x, start);
    while (next->n) {
        cand_t c = next->e[0];
        if ((-c.d) > radius && top->n == top_limit)
            break;
        heap_pop(next);
        x->st.base_pops++;
        uint32_t n = x->cnt0[c.s], i;
        const uint32_t* l = x->nbr0 + (size_t)c.s * x->M0;
        for (i = 0; i < n; ++i) {
            uint32_t s = l[i];
            if (visits_set(x, s))
                continue;
            x->st.visited_members++;
            float d = measure_qv(x, q, s);
            if (top->n < top_limit || d < radius) {
                heap_push(next, -d, s);
                if (x->keys[s] == UINT64_MAX) /* predicate key != free_key_, index_dense.hpp:1448 */
                    continue;
                sbuf_insert(top, d, s, top_limit);
                radius = top->e[top->n - 1].d;
            }
        }
    }
}

/* The beam of search_base / search_to_insert with the CUDA engine's queue discipline (lantern_b200/csrc/walk.cuh
 * beam_impl), for search (level 0, skip == UINT32_MAX) and for insertion (level l, skip == the new node) alike: the
 * candidate queue is the set of unexpanded entries of `top` (closest first; among equal distances the most recently
 * inserted first, which is what insert-before-equal gives) plus a LIFO "limbo" of unexpanded entries evicted at exactly
 * the current radius (at most 64, walk.cuh kLimboCap; dropped when the radius shrinks below them).  A popped `skip` is
 * not expanded (index.hpp:3357; beam_impl's `c == skip`).  Identical to the heap beams whenever no two candidate
 * distances are exactly equal; with ties only the ORDER of equal-distance expansions differs from the reference's binary
 * heap, and then this order is the engine's: its searches and its builds are pinned against this function. */
static void beam_engine_order(ora_index* x, const void* q, uint32_t start, uint32_t skip, int level, size_t top_limit) {
    cvec_t* top = &x->top;
    uint8_t* expanded = (uint8_t*)calloc(top_limit + 1, 1);
    uint32_t limbo[64];
    size_t limbo_n = 0, i;
    float limbo_d = 0.f;
    visits_clear(x);
    top->n = 0;
    cvec_reserve(top, top_limit + 1);
    float radius = measure_qv(x, q, start);
    top->e[0].d = radius, top->e[0].s = start, top->n = 1;
    visits_set(x, start);
    for (;;) {
        uint32_t c = UINT32_MAX;
        for (i = 0; i < top->n; ++i)
            if (!expanded[i]) {
                c = top->e[i].s, expanded[i] = 1;
                break;
            }
        if (c == UINT32_MAX && limbo_n)
            c = limbo[--limbo_n];
        if (c == UINT32_MAX)
            break;
        if (c == skip)
            continue;
        if (skip == UINT32_MAX) /* search: counted like search_base */
            x->st.base_pops++;
        uint32_t* cnt;
        const uint32_t* l = nbr_list(x, c, level, &cnt);
        uint32_t n = *cnt, j;
        for (j = 0; j < n; ++j) {
            uint32_t s = l[j];
            if (visits_set(x, s))
                continue;
            x->st.visited_members++;
            float d = measure_qv(x, q, s);
            if (top->n < top_limit || d < top->e[top->n - 1].d) {
                size_t pos = sbuf_lower_bound(top, d), full = (top->n == top_limit);
                float ev_d = 0.f;
                uint32_t ev_s = UINT32_MAX;
                int ev_expanded = 1;
                if (full)
                    ev_d = top->e[top_limit - 1].d, ev_s = top->e[top_limit - 1].s, ev_expanded = expanded[top_limit - 1];
                size_t last = full ? top_limit - 1 : top->n;
                memmove(top->e + pos + 1, top->e + pos, (last - pos) * sizeof(cand_t));
                memmove(expanded + pos + 1, expanded + pos, last - pos);
                top->e[pos].d = d, top->e[pos].s = s, expanded[pos] = 0;
                top->n = last + 1;
                radius = top->e[top->n - 1].d;
                if (limbo_n && radius < limbo_d)
                    limbo_n = 0;
                if (ev_s != UINT32_MAX && !ev_expanded && ev_d == radius && limbo_n < 64)
                    limbo[limbo_n++] = ev_s, limbo_d = radius;
            }
        }
    }
    free(expanded);
}

/* search_to_insert_, index.hpp:3324-3392 (engine_order: the engine's tie order, beam_engine_order). */
static void search_to_insert(ora_index* x, const void* q, uint32_t start, uint32_t new_slot, int level,
                             size_t top_limit) {
    if (x->engine_order) {
        beam_engine_order(x, q, start, new_slot, level, top_limit);
        return;
    }
    cvec_t *next = &x->next, *top = &x->top;
    visits_clear(x);
    next->n = 0, top->n = 0;
    float radius = measure_qv(x, q, start);
    heap_push(next, -radius, start);
    sbuf_insert_reserved(top, radius, start);
    visits_set(x, start);
    while (next->n) {
        cand_t c = next->e[0];
        if ((-c.d) > radius && top->n == top_limit)
            break;
        heap_pop(next);
        if (c.s == new_slot)
            continue;
        uint32_t* cnt;
        uint32_t* l = nbr_list(x, c.s, level, &cnt);
        uint32_t n = *cnt, i;
        for (i = 0; i < n; ++i) {
            uint32_t s = l[i];
            if (visits_set(x, s))
                continue;
            x->st.visited_members++;
            float d = measure_qv(x, q, s);
            if (top->n < top_limit || d < radius) {
                heap_push(next, -d, s);
                sbuf_insert(top, d, s, top_limit);
                radius = top->e[top->n - 1].d;
            }
        }
    }
}

/* refine_, index.hpp:3515-3561, with skip_pruned_connections == false (index.hpp:1245): the
 * selected prefix is followed by whatever sits at positions [submitted, needed) -- stale
 * entries, possibly duplicates of selected ones.  Returns the size of the resulting view. */
static size_t refine(ora_index* x, size_t needed) {
    cvec_t* top = &x->top;
    size_t count = top->n;
    if (count < needed)
        return count;
    size_t submitted = 1, consumed = 1;
    while (submitted < needed && consumed < count) {
        cand_t c = top->e[consumed];
        int good = 1;
        size_t i;
        for (i = 0; i < submitted; ++i) {
            float inter = measure_vv(x, c.s, top->e[i].s);
            if (inter < c.d) {
                good = 0;
                break;
            }
        }
        if (good) {
            top->e[submitted] = top->e[consumed];
            submitted++;
        }
        consumed++;
    }
    size_t keep = submitted > needed ? submitted : needed;
    if (keep < top->n)
        top->n = keep;
    return top->n;
}

/* choose_random_level_, index.hpp:3208-3212, with libstdc++'s std::default_random_engine
 * (minstd_rand0: x <- 16807 x mod 2^31-1, seed 1) and uniform_real_distribution<double>
 * (generate_canonical<double,53>: two draws, sum = (x1-1) + (x2-1)*R, R = 2147483646). */
static uint32_t minstd_next(uint32_t* s) {
    *s = (uint32_t)(((uint64_t)*s * 16807ull) % 2147483647ull);
    return *s;
}
static int16_t choose_random_level(uint32_t* rng, size_t M) {
    const double R = 2147483646.0;
    double sum = (double)(minstd_next(rng) - 1u);
    sum += (double)(minstd_next(rng) - 1u) * R;
    double u = sum / (R * R);
    if (u >= 1.0)
        u = nextafter(1.0, 0.0);
    double r = -log(u) * (1.0 / log((double)M));
    return (int16_t)r;
}

int ora_level_sequence(size_t connectivity, size_t count, int16_t* out) {
    uint32_t rng = 1u;
    size_t i;
    for (i = 0; i < count; ++i)
        out[i] = choose_random_level(&rng, connectivity);
    return 0;
}

/* Casting of an incoming vector to the metric's scalar kind: index_dense.hpp:1404-1410,1435-1441. */
static const void* cast_input(ora_index* x, const void* v, int kind) {
    if (kind == ORA_F32 && x->quant != ORA_F32) {
        ora_cast_f32((const float*)v, x->dims, x->quant, x->cast_buf);
        return x->cast_buf;
    }
    return v; /* f32->f32 and b1->b1: no cast (index_plugins.hpp:889-907) */
}

/* index_gt::add, index.hpp:2479-2564 + connect_node_across_levels_ :3119-3136 +
 * connect_new_node_ :3139-3160 + reconnect_neighbor_nodes_ :3163-3206. */
int ora_add(ora_index* x, uint64_t key, const void* vector, int kind, int level, ora_stats* stats) {
    if (x->n >= x->cap)
        return -1; /* "Reserve capacity ahead of insertions!" index.hpp:2514-2517 */
    memset(&x->st, 0, sizeof(x->st));
    const void* value = cast_input(x, vector, kind);
    /* the generator is only advanced when no level is supplied (index.hpp:2509) */
    int target = level >= 0 ? level : choose_random_level(&x->rng, x->M);
    uint32_t slot = (uint32_t)x->n;
    x->n++;
    x->keys[slot] = key;
    x->levels[slot] = (int16_t)target;
    x->cnt0[slot] = 0;
    memset(x->nbr0 + (size_t)slot * x->M0, 0, x->M0 * sizeof(uint32_t));
    x->upper[slot] = target > 0 ? (uint32_t*)calloc((size_t)target * (1 + x->M), sizeof(uint32_t)) : NULL;
    /* on_success callback -> set_vector_at (index_dense.hpp:1415-1417; pq: compress, lantern_storage.hpp:442-443) */
    if (x->pq)
        ora_pq_compress(x->codebook, x->dims, x->ncent, x->nsub, (const float*)value,
                        x->vectors + (size_t)slot * x->stored_bytes, x->compat128);
    else
        memcpy(x->vectors + (size_t)slot * x->stored_bytes, value, x->stored_bytes);

    if (slot == 0) {
        x->entry = 0, x->max_level = target;
        if (stats)
            *stats = x->st;
        return 0;
    }
    int max_level = x->max_level;
    uint32_t closest = search_for_one(x, value, (uint32_t)x->entry, max_level, target);
    int l;
    for (l = target < max_level ? target : max_level; l >= 0; --l) {
        search_to_insert(x, value, closest, slot, l, x->efc);
        /* connect_new_node_: refine to `connectivity` on EVERY level, base included (:3149) */
        size_t view = refine(x, x->M), i;
        uint32_t* cnt;
        uint32_t* mine = nbr_list(x, slot, l, &cnt);
        for (i = 0; i < view; ++i)
            mine[(*cnt)++] = x->top.e[i].s;
        closest = mine[0];
        /* reconnect_neighbor_nodes_ */
        size_t cmax = l ? x->M : x->M0;
        uint32_t mine_n = *cnt, j;
        uint32_t mine_copy[512];
        memcpy(mine_copy, mine, mine_n * sizeof(uint32_t));
        for (j = 0; j < mine_n; ++j) {
            uint32_t close = mine_copy[j];
            if (close == slot)
                continue;
            uint32_t* ccnt;
            uint32_t* cl = nbr_list(x, close, l, &ccnt);
            if (*ccnt < cmax) {
                cl[(*ccnt)++] = slot;
                continue;
            }
            x->top.n = 0;
            sbuf_insert_reserved(&x->top, measure_qv(x, value, close), slot);
            uint32_t k;
            for (k = 0; k < *ccnt; ++k)
                sbuf_insert_reserved(&x->top, measure_vv(x, close, cl[k]), cl[k]);
            memset(cl, 0, *ccnt * sizeof(uint32_t)); /* neighbors_ref_t::clear zeroes the list, :1777-1781 */
            *ccnt = 0;
            size_t v2 = refine(x, cmax), t;
            for (t = 0; t < v2; ++t)
                cl[(*ccnt)++] = x->top.e[t].s;
        }
    }
    if (target > max_level)
        x->entry = slot, x->max_level = target;
    if (stats)
        *stats = x->st;
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * Model of the CUDA engine's BATCHED build (lantern_b200/csrc/build.cu) -- not a reference function.
 * The reference inserts one node at a time; the engine inserts batches in two phases so that thousands of inserts
 * run concurrently.  This restates that schedule on top of the reference procedures above, so that the engine's
 * default build can be checked bit for bit against a CPU specification (tests/test_gpu_build_model.py, with engine_order on
 * so that the insertion beams break distance ties as the engine does) instead of only statistically (recall):
 *   levels are drawn up front for all pending vectors (same generator, same order as sequential inserts);
 *   a batch holds min(remaining, batch_cap, max(1, visible / build_ratio)) nodes and is cut in front of a node whose
 *   level exceeds the current top level (such a node is inserted alone and then becomes the entry point);
 *   phase 1, per node of the batch, all against the graph as it was BEFORE the batch: greedy descent, efc-wide beam
 *   and heuristic per level (search_to_insert + refine, exactly as in ora_add), own lists written, one reverse-link
 *   request (level, target, distance, new node) per selected neighbour;
 *   phase 2: requests grouped by (level, target) in (node, position) order -- a stable sort, as the radix sort of the
 *   engine is -- and applied one after the other: append while the list has room, else re-prune {new} + list with the
 *   heuristic.  Distances target->neighbour are measured once per group, when it first overflows; entries kept by a
 *   re-prune carry their distance to the next request of the same group.
 * With batch_cap == 1 this is ora_add (byte-identical index file; tests/test_oracle_ref.py).  PQ indexes are not
 * modelled (a carried distance of a new node is value-vs-stored there, a re-measured one stored-vs-stored).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    uint64_t key; /* (level << 32) | target */
    float d;
    uint32_t u;
} req_t;

static void reqs_stable_sort(req_t* a, req_t* tmp, size_t n) { /* bottom-up merge sort by key: stable */
    size_t w, i;
    for (w = 1; w < n; w *= 2) {
        for (i = 0; i < n; i += 2 * w) {
            size_t l = i, m = i + w < n ? i + w : n, r = i + 2 * w < n ? i + 2 * w : n, a0 = l, b0 = m, o = l;
            while (a0 < m && b0 < r)
                tmp[o++] = a[b0].key < a[a0].key ? a[b0++] : a[a0++];
            while (a0 < m)
                tmp[o++] = a[a0++];
            while (b0 < r)
                tmp[o++] = a[b0++];
        }
        memcpy(a, tmp, n * sizeof(req_t));
    }
}

int ora_add_batch_engine(ora_index* x, const uint64_t* keys, const void* vectors, size_t n, size_t stride, int kind,
                         size_t batch_cap, size_t build_ratio) {
    if (x->pq)
        return -2;
    if (x->n + n > x->cap)
        return -1;
    if (!n)
        return 0;
    if (!batch_cap)
        batch_cap = 1;
    if (!build_ratio)
        build_ratio = 1;
    const size_t n0 = x->n, P = n, M = x->M, M0 = x->M0;
    size_t i, pos = 0;
    /* node records of all pending vectors: the engine stores them at insertion ids n0.. before the first batch */
    for (i = 0; i < P; ++i) {
        const size_t slot = n0 + i;
        const void* value = cast_input(x, (const uint8_t*)vectors + i * stride, kind);
        int target = choose_random_level(&x->rng, M);
        x->keys[slot] = keys[i];
        x->levels[slot] = (int16_t)target;
        x->cnt0[slot] = 0;
        memset(x->nbr0 + slot * M0, 0, M0 * sizeof(uint32_t));
        x->upper[slot] = target > 0 ? (uint32_t*)calloc((size_t)target * (1 + M), sizeof(uint32_t)) : NULL;
        memcpy(x->vectors + slot * x->stored_bytes, value, x->stored_bytes);
    }
    x->n = n0 + P; /* records exist (ora_free walks them); visibility is governed by entry / links below */
    size_t visible = n0;
    if (n0 == 0) { /* first node: entry point, no links (index.hpp:2538-2543) */
        x->entry = 0, x->max_level = x->levels[0];
        visible = 1, pos = 1;
    }
    req_t *reqs = NULL, *tmp = NULL;
    size_t reqs_cap = 0;
    float* dist = (float*)malloc((M0 + 2) * sizeof(float));
    while (pos < P) {
        size_t bsz = 1;
        if (x->levels[n0 + pos] <= x->max_level) {
            size_t ramp = visible / build_ratio;
            if (ramp < 1)
                ramp = 1;
            bsz = P - pos;
            if (bsz > batch_cap)
                bsz = batch_cap;
            if (bsz > ramp)
                bsz = ramp;
            for (i = 1; i < bsz; ++i)
                if (x->levels[n0 + pos + i] > x->max_level) {
                    bsz = i;
                    break;
                }
        }
        const int max_level = x->max_level;
        const uint32_t entry = (uint32_t)x->entry;
        const size_t need = bsz * M * (size_t)(max_level + 1);
        if (need > reqs_cap) {
            reqs_cap = need * 2;
            reqs = (req_t*)realloc(reqs, reqs_cap * sizeof(req_t));
            tmp = (req_t*)realloc(tmp, reqs_cap * sizeof(req_t));
        }
        size_t nreq = 0, b;
        /* ---- phase 1: every node of the batch against the graph before the batch ---- */
        for (b = 0; b < bsz; ++b) {
            const uint32_t slot = (uint32_t)(n0 + pos + b);
            const int lu = x->levels[slot];
            const void* value = x->vectors + (size_t)slot * x->stored_bytes; /* cast value == stored vector (no pq) */
            uint32_t closest = search_for_one(x, value, entry, max_level, lu);
            int l;
            for (l = lu < max_level ? lu : max_level; l >= 0; --l) {
                search_to_insert(x, value, closest, slot, l, x->efc);
                size_t view = refine(x, M), t;
                uint32_t* cnt;
                uint32_t* mine = nbr_list(x, slot, l, &cnt);
                for (t = 0; t < view; ++t) {
                    mine[(*cnt)++] = x->top.e[t].s;
                    reqs[nreq].key = ((uint64_t)(uint32_t)l << 32) | x->top.e[t].s;
                    reqs[nreq].d = x->top.e[t].d, reqs[nreq].u = slot;
                    nreq++;
                }
                closest = mine[0];
            }
        }
        /* ---- phase 2: reverse links, grouped by (level, target), in (node, position) order ---- */
        reqs_stable_sort(reqs, tmp, nreq);
        size_t r = 0;
        while (r < nreq) {
            const uint64_t key = reqs[r].key;
            const int level = (int)(key >> 32);
            const uint32_t v = (uint32_t)key;
            const size_t cmax = level ? M : M0;
            uint32_t* ccnt;
            uint32_t* cl = nbr_list(x, v, level, &ccnt);
            int have_d = 0;
            for (; r < nreq && reqs[r].key == key; ++r) {
                const uint32_t u = reqs[r].u;
                const float d_uv = reqs[r].d;
                uint32_t k;
                if (*ccnt < cmax) { /* index.hpp:3186-3189 */
                    dist[*ccnt] = d_uv;
                    cl[(*ccnt)++] = u;
                    continue;
                }
                if (!have_d) { /* distances target -> each current neighbour (index.hpp:3196-3198) */
                    for (k = 0; k < *ccnt; ++k)
                        dist[k] = measure_vv(x, v, cl[k]);
                    have_d = 1;
                }
                x->top.n = 0;
                sbuf_insert_reserved(&x->top, d_uv, u);
                for (k = 0; k < *ccnt; ++k)
                    sbuf_insert_reserved(&x->top, dist[k], cl[k]);
                memset(cl, 0, *ccnt * sizeof(uint32_t));
                *ccnt = 0;
                size_t v2 = refine(x, cmax), t;
                for (t = 0; t < v2; ++t) {
                    dist[*ccnt] = x->top.e[t].d;
                    cl[(*ccnt)++] = x->top.e[t].s;
                }
            }
        }
        visible += bsz;
        if (x->levels[n0 + pos] > x->max_level) { /* index.hpp:2558-2562 */
            x->entry = n0 + pos;
            x->max_level = x->levels[n0 + pos];
        }
        pos += bsz;
    }
    free(reqs), free(tmp), free(dist);
    return 0;
}

/* index_gt::search, index.hpp:2680-2730. */
size_t ora_search(ora_index* x, const void* query, int kind, size_t k, size_t ef, uint64_t* keys, float* distances,
                  ora_stats* stats) {
    memset(&x->st, 0, sizeof(x->st));
    if (!x->n) {
        if (stats)
            *stats = x->st;
        return 0;
    }
    const void* q = cast_input(x, query, kind);
    size_t expansion = ef ? ef : x->ef;
    if (expansion < k)
        expansion = k;
    uint32_t closest = search_for_one(x, q, (uint32_t)x->entry, x->max_level, 0);
    if (x->engine_order)
        beam_engine_order(x, q, closest, UINT32_MAX, 0, expansion);
    else
        search_base(x, q, closest, expansion);
    size_t found = x->top.n < k ? x->top.n : k, i;
    for (i = 0; i < found; ++i) {
        keys[i] = x->keys[x->top.e[i].s];
        distances[i] = x->top.e[i].d;
    }
    if (stats)
        *stats = x->st;
    return found;
}

/* ------------------------------------------------------------------------------------------
 * File format.  index_dense.hpp:42-79 (80-byte head), index.hpp:1696-1703 (40-byte header),
 * lantern_storage.hpp:486-521 (u64 vector_size_bytes, u64 node_count, then per node the tape
 * [key u64][level i16][u32 cnt + M0 x uint48][level x (u32 cnt + M x uint48)] followed by the
 * vector bytes / PQ codes, no padding).  Verified byte-for-byte against oracle/_ref.
 * ---------------------------------------------------------------------------------------- */
static uint8_t metric_char(int m) {
    switch (m) {
    case ORA_METRIC_COS: return 'c';
    case ORA_METRIC_IP: return 'i';
    case ORA_METRIC_L2SQ: return 'e';
    case ORA_METRIC_HAMMING: return 'b';
    default: return 0;
    }
}
static uint8_t scalar_code(int k) { /* scalar_kind_t, index_plugins.hpp:130-152 */
    switch (k) {
    case ORA_B1: return 1;
    case ORA_F64: return 4;
    case ORA_F32: return 5;
    case ORA_F16: return 6;
    case ORA_I8: return 15;
    default: return 0;
    }
}

size_t ora_serialized_length(const ora_index* x) {
    size_t total = 136, i;
    for (i = 0; i < x->n; ++i)
        total += 10 + (4 + 6 * x->M0) + (size_t)x->levels[i] * (4 + 6 * x->M) + x->stored_bytes;
    return total;
}

static uint8_t* put_u64(uint8_t* p, uint64_t v) {
    memcpy(p, &v, 8);
    return p + 8;
}
static uint8_t* put_list(uint8_t* p, const uint32_t* ids, uint32_t cnt, size_t width) {
    size_t i;
    memcpy(p, &cnt, 4);
    p += 4;
    memset(p, 0, 6 * width);
    for (i = 0; i < cnt; ++i) {
        uint64_t v = ids[i];
        memcpy(p + 6 * i, &v, 6);
    }
    return p + 6 * width;
}

size_t ora_save_buffer(const ora_index* x, void* buffer, size_t length) {
    size_t need = ora_serialized_length(x), i;
    if (length < need)
        return 0;
    uint8_t* p = (uint8_t*)buffer;
    memset(p, 0, 80);
    memcpy(p, "usearch", 7);
    uint16_t ver[3] = {2, 8, 14};
    memcpy(p + 7, ver, 6);
    p[13] = metric_char(x->metric), p[14] = scalar_code(x->quant), p[15] = 8, p[16] = 16;
    uint64_t v = x->n;
    memcpy(p + 17, &v, 8);
    v = 0;
    memcpy(p + 25, &v, 8);
    v = x->dims;
    memcpy(p + 33, &v, 8);
    p[41] = 0;
    p += 80;
    p = put_u64(p, x->n), p = put_u64(p, x->M), p = put_u64(p, x->M0);
    p = put_u64(p, (uint64_t)(x->max_level < 0 ? 0 : x->max_level)), p = put_u64(p, x->entry);
    p = put_u64(p, x->vec_bytes), p = put_u64(p, x->n);
    for (i = 0; i < x->n; ++i) {
        int l;
        p = put_u64(p, x->keys[i]);
        memcpy(p, &x->levels[i], 2);
        p += 2;
        p = put_list(p, x->nbr0 + i * x->M0, x->cnt0[i], x->M0);
        for (l = 1; l <= x->levels[i]; ++l) {
            uint32_t* base = x->upper[i] + (size_t)(l - 1) * (1 + x->M);
            p = put_list(p, base + 1, base[0], x->M);
        }
        memcpy(p, x->vectors + i * x->stored_bytes, x->stored_bytes);
        p += x->stored_bytes;
    }
    return (size_t)(p - (uint8_t*)buffer);
}

int ora_load_buffer(ora_index* x, const void* buffer, size_t length) {
    const uint8_t* p = (const uint8_t*)buffer;
    if (length < 136 || memcmp(p, "usearch", 7) != 0)
        return -1;
    uint64_t hdr[7];
    memcpy(hdr, p + 80, 56);
    size_t n = hdr[0], i;
    if (hdr[1] != x->M || hdr[2] != x->M0)
        return -2;
    if (!ora_reserve(x, n ? n : 1))
        return -3;
    for (i = 0; i < x->n; ++i)
        free(x->upper[i]), x->upper[i] = NULL;
    x->n = 0;
    const uint8_t* end = p + length;
    p += 136;
    for (i = 0; i < n; ++i) {
        int16_t level;
        int l;
        uint32_t cnt, j;
        if (p + 10 > end)
            return -4;
        memcpy(&x->keys[i], p, 8);
        memcpy(&level, p + 8, 2);
        p += 10;
        x->levels[i] = level;
        size_t tape = (4 + 6 * x->M0) + (size_t)level * (4 + 6 * x->M) + x->stored_bytes;
        if (p + tape > end)
            return -4;
        memcpy(&cnt, p, 4);
        x->cnt0[i] = cnt;
        for (j = 0; j < x->M0; ++j) {
            uint64_t v = 0;
            memcpy(&v, p + 4 + 6 * j, 6);
            x->nbr0[i * x->M0 + j] = (uint32_t)v;
        }
        p += 4 + 6 * x->M0;
        x->upper[i] = level > 0 ? (uint32_t*)calloc((size_t)level * (1 + x->M), sizeof(uint32_t)) : NULL;
        for (l = 1; l <= level; ++l) {
            uint32_t* base = x->upper[i] + (size_t)(l - 1) * (1 + x->M);
            memcpy(&cnt, p, 4);
            base[0] = cnt;
            for (j = 0; j < x->M; ++j) {
                uint64_t v = 0;
                memcpy(&v, p + 4 + 6 * j, 6);
                base[1 + j] = (uint32_t)v;
            }
            p += 4 + 6 * x->M;
        }
        memcpy(x->vectors + i * x->stored_bytes, p, x->stored_bytes);
        p += x->stored_bytes;
        x->n = i + 1;
    }
    x->max_level = n ? (int)hdr[3] : -1;
    x->entry = hdr[4];
    return 0;
}

/* exact_search_t, index_plugins.hpp:1582-1675: all distances, k smallest ascending.
 * Ties are broken by lower offset here (the reference's partial_sort is unspecified among ties). */
void ora_exact_search(const void* dataset, size_t n, size_t dataset_stride, const void* queries, size_t nq,
                      size_t queries_stride, int kind, size_t dims, int metric, size_t k, uint64_t* keys,
                      float* distances) {
    size_t q, i;
    cvec_t top = {0, 0, 0};
    for (q = 0; q < nq; ++q) {
        const uint8_t* qp = (const uint8_t*)queries + q * queries_stride;
        top.n = 0;
        for (i = 0; i < n; ++i) {
            /* metric(dataset, query) argument order as in index_plugins.hpp:1630 */
            float d = ora_distance((const uint8_t*)dataset + i * dataset_stride, qp, kind, dims, metric);
            /* stable: insert AFTER equal elements -> upper bound */
            size_t lo = 0, hi = top.n;
            while (lo < hi) {
                size_t mid = lo + (hi - lo) / 2;
                if (top.e[mid].d <= d)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            if (lo >= k)
                continue;
            cvec_reserve(&top, top.n + 1);
            size_t full = (top.n == k);
            memmove(top.e + lo + 1, top.e + lo, (top.n - lo - full) * sizeof(cand_t));
            top.e[lo].d = d, top.e[lo].s = (uint32_t)i;
            top.n += !full;
        }
        for (i = 0; i < k; ++i) {
            keys[q * k + i] = i < top.n ? top.e[i].s : UINT64_MAX;
            distances[q * k + i] = i < top.n ? top.e[i].d : INFINITY;
        }
    }
    free(top.e);
}

/* ------------------------------------------------------------------------------------------
 * PQ codebook training.  Restates lantern_hnsw/src/hnsw/product_quantization.c:51-293 (k distinct dataset rows as
 * initial centres; assign by usearch_distance with strict '<'; centre = float mean of its members, empty clusters keep
 * their centre; stop when mean_c distance(old_c, new_c) <= 0.1 or after max_iter rounds; one k-means per subvector).
 * PARITY PINNED: the reference file itself is compiled unmodified into oracle/_ref/liboracle_refpq.so (oracle/Makefile
 * target refpq, stand-in postgres.h in oracle/pg_shim/, PRNG scripted) and this function reproduces its codebooks bit for
 * bit (tests/test_oracle_ref.py::test_kmeans_restatement_equals_the_reference).  The initial rows are an INPUT here
 * (init_rows[nsub][ncent]): in the reference they come from libc/Postgres' PRNG.
 * ---------------------------------------------------------------------------------------- */
int ora_kmeans(const float* data, size_t n, size_t dims, size_t nsub, size_t ncent, int metric, size_t max_iter,
               const uint32_t* init_rows, float* codebook) {
    size_t sd = dims / nsub, s, c, i, j, it;
    uint32_t* assign = (uint32_t*)malloc(n * sizeof(uint32_t));
    float* old = (float*)malloc(ncent * sd * sizeof(float));
    float* sum = (float*)malloc(sd * sizeof(float));
    int rounds = 0;
    for (s = 0; s < nsub; ++s) {
        for (c = 0; c < ncent; ++c)
            memcpy(codebook + c * dims + s * sd, data + (size_t)init_rows[s * ncent + c] * dims + s * sd, sd * sizeof(float));
        for (it = 0; it < max_iter; ++it) {
            if ((int)(it + 1) > rounds)
                rounds = (int)(it + 1);
            for (i = 0; i < n; ++i) {
                float best = 3.402823466e+38f;
                uint32_t bc = 0;
                for (c = 0; c < ncent; ++c) {
                    float d = ora_distance(data + i * dims + s * sd, codebook + c * dims + s * sd, ORA_F32, sd, metric);
                    if (d < best)
                        best = d, bc = (uint32_t)c;
                }
                assign[i] = bc;
            }
            float shift = 0.f;
            for (c = 0; c < ncent; ++c) {
                size_t cnt = 0;
                memcpy(old + c * sd, codebook + c * dims + s * sd, sd * sizeof(float));
                memset(sum, 0, sd * sizeof(float));
                for (i = 0; i < n; ++i)
                    if (assign[i] == c) {
                        for (j = 0; j < sd; ++j)
                            sum[j] += data[i * dims + s * sd + j];
                        cnt++;
                    }
                if (cnt)
                    for (j = 0; j < sd; ++j)
                        codebook[c * dims + s * sd + j] = sum[j] / (float)cnt;
                shift += ora_distance(old + c * sd, codebook + c * dims + s * sd, ORA_F32, sd, metric);
            }
            if (shift / (float)ncent <= 0.1f)
                break;
        }
    }
    free(assign), free(old), free(sum);
    return rounds;
}
