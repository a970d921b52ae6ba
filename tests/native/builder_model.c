/*
 *  tests/native/builder_model.c — the batch schedule of the GPU builder (usearch_b200/csrc/builder.cu, DESIGN.md §3.5)
 *  restated on the host, one decision at a time, so that a GPU-built graph can be compared with it list for list.
 *
 *  The containers (`next` heap, `top` sorted buffer, visits set), the blob parser and the pinned metrics are the port's
 *  (oracle/hnsw_oracle.c, included unchanged through port_f64.c, which adds the f64 metric of f64_pinned.h). What is
 *  restated here is what the builder does with them:
 *
 *    add          reused slots first, in batches of min(left, cap, max(n / ratio, 1)) that are never cut; then the
 *                 appended slots: the first member of an empty graph becomes the entry point with no links, and every
 *                 other batch has min(left, cap, max(n / ratio, 1)) members and ends right after the first member
 *                 above the top level. `n` counts the slots linked so far.
 *    tasks        level 0 of every member of the batch, then levels 1..min(level, top) member by member
 *    search       per task: search_for_one_ (index.hpp:3963-4003) from the entry point down to level + 1, then
 *                 search_to_insert_ (:4010-4079) on the level with ef = expansion_add, both over the graph as it stood
 *                 before the batch; a reused member's own slot never enters its own `top` (search_to_update_, :4086-4168)
 *    forward      candidates cut to min(count, ef, 256); refine_ (:4276-4318) with needed = M on every level (fewer
 *                 candidates than needed: all kept, ascending); the member's row is written with an EMPTY_SLOT tail
 *    pairs        (level, neighbour, member, d(member, neighbour)) at index task * M + rank, grouped by (level, neighbour)
 *                 in index order
 *    reverse      per (level, neighbour): the run is cut to its first 256 - listed arrivals, then arrivals the row
 *                 already holds are dropped; the rest are appended if they fit, otherwise the listed entries get
 *                 d(neighbour, s), the arrivals keep their forward distance, everything is sorted ascending with ties
 *                 broken by slot, and refine_ keeps up to the level's capacity
 *    after        the entry point and the top level move to the batch's member above the top level, if any
 *
 *  Build: cc -O2 -ffp-contract=off -shared -fPIC builder_model.c -lm -lpthread (tests/builder_model.py does it).
 */
#include "port_f64.c"

#define BM_EMPTY 0xFFFFFFFFu
#define BM_CAND_MAX 256u /* what one refine holds on the GPU (LINK_CAND_MAX) */

enum { BM_BATCHES, BM_TASKS, BM_REVERSE_RUNS, BM_REVERSE_REFINES, BM_REVERSE_REFINES_BASE, BM_ROOM_CUTS, BM_CANDIDATE_CUTS,
       BM_SHORT_REFINES, BM_SORT_TIES, BM_REUSED, BM_HELD_ARRIVALS, BM_COUNTERS };

typedef struct {
    uint8_t metric_kind, scalar_kind;
    size_t dims, bytes_per_vector, third;
    oracle_metric_t metric;
    size_t m, m0;
    size_t size, capacity; /* slots stored */
    size_t linked;         /* slots [0, linked) are in the graph (the device's `d.n`) */
    uint8_t* vectors;
    uint64_t* keys;
    int16_t* levels;
    int32_t* linked_in;  /* per slot: the batch that linked it (-1: it came with the starting graph) */
    int32_t* written_in; /* per slot: the last batch that wrote one of its rows */
    uint32_t** rows; /* per slot: m0 entries of level 0, then m per upper level; EMPTY_SLOT tails */
    uint32_t entry;
    int max_level;
    uint64_t counters[BM_COUNTERS];
    context_t ctx;
} bm_index_t;

static oracle_metric_t bm_pick_metric(uint8_t metric, uint8_t scalar) {
    if (scalar == SK_F64) return metric == 'e' ? wrap_l2sq_f64 : metric == 'i' ? wrap_ip_f64 : metric == 'c' ? wrap_cos_f64 : NULL;
    return pick_metric(metric, scalar);
}

static uint32_t* bm_row(bm_index_t const* b, uint32_t slot, size_t level) {
    return b->rows[slot] + (level ? b->m0 + (level - 1) * b->m : 0);
}
static size_t bm_capacity_of(bm_index_t const* b, size_t level) { return level ? b->m : b->m0; }
static size_t bm_listed(bm_index_t const* b, uint32_t slot, size_t level) {
    uint32_t const* row = bm_row(b, slot, level);
    size_t n = 0, cap = bm_capacity_of(b, level);
    while (n < cap && row[n] != BM_EMPTY) ++n;
    return n;
}
static uint8_t const* bm_vec(bm_index_t const* b, uint32_t slot) { return b->vectors + (size_t)slot * b->bytes_per_vector; }
static float bm_measure(bm_index_t* b, void const* q, uint32_t slot) {
    b->ctx.computed_distances++;
    return b->metric(q, bm_vec(b, slot), b->third);
}

static int bm_reserve(bm_index_t* b, size_t slots) {
    if (slots <= b->capacity) return 1;
    size_t cap = b->capacity ? b->capacity : 16;
    while (cap < slots) cap *= 2;
    uint8_t* v = (uint8_t*)realloc(b->vectors, cap * b->bytes_per_vector + 1);
    if (!v) return 0;
    b->vectors = v;
    uint64_t* k = (uint64_t*)realloc(b->keys, cap * 8);
    if (!k) return 0;
    b->keys = k;
    int16_t* l = (int16_t*)realloc(b->levels, cap * 2);
    if (!l) return 0;
    b->levels = l;
    int32_t* li = (int32_t*)realloc(b->linked_in, cap * 4);
    if (!li) return 0;
    b->linked_in = li;
    int32_t* wi = (int32_t*)realloc(b->written_in, cap * 4);
    if (!wi) return 0;
    b->written_in = wi;
    uint32_t** r = (uint32_t**)realloc(b->rows, cap * sizeof(uint32_t*));
    if (!r) return 0;
    b->rows = r;
    b->capacity = cap;
    return 1;
}

static int bm_alloc_rows(bm_index_t* b, uint32_t slot, int level) {
    size_t const n = b->m0 + (size_t)level * b->m;
    b->rows[slot] = (uint32_t*)malloc(n * 4 + 4);
    if (!b->rows[slot]) return 0;
    memset(b->rows[slot], 0xFF, n * 4);
    return 1;
}

bm_index_t* bm_new(int metric_kind, int scalar_kind, size_t dims, size_t m, size_t m0) {
    bm_index_t* b = (bm_index_t*)calloc(1, sizeof(bm_index_t));
    if (!b) return NULL;
    b->metric_kind = (uint8_t)metric_kind;
    b->scalar_kind = (uint8_t)scalar_kind;
    b->metric = bm_pick_metric(b->metric_kind, b->scalar_kind);
    if (!b->metric || m < 2 || m0 < m) { free(b); return NULL; }
    b->dims = dims;
    b->bytes_per_vector = (dims * bits_per_scalar(b->scalar_kind) + 7) / 8;
    b->third = b->scalar_kind == SK_B1 ? (dims + 7) / 8 : dims;
    b->m = m;
    b->m0 = m0;
    return b;
}

void bm_free(bm_index_t* b) {
    if (!b) return;
    for (size_t i = 0; i < b->size; ++i) free(b->rows[i]);
    free(b->rows);
    free(b->vectors);
    free(b->keys);
    free(b->levels);
    free(b->linked_in);
    free(b->written_in);
    context_free(&b->ctx);
    free(b);
}

/* the graph of a v2 blob: every slot is linked */
bm_index_t* bm_open(void const* blob, size_t length, char const** error) {
    *error = NULL;
    uint8_t const* p = (uint8_t const*)blob;
    if (length < 8 + 64 + 40) { *error = "File is corrupted and lacks matrix dimensions"; return NULL; }
    uint64_t const head = 8 + (uint64_t)rd_u32(p) * rd_u32(p + 4);
    if (head + 64 > length) { *error = "File is corrupted and lacks a header"; return NULL; }
    int const f64 = p[head + 14] == SK_F64;
    oracle_index_t* ix = f64 ? oracle_open_f64(blob, length, error) : oracle_open(blob, length, error);
    if (!ix) return NULL;
    bm_index_t* b = bm_new(ix->metric_kind, ix->scalar_kind, ix->dimensions, ix->connectivity, ix->connectivity_base);
    if (!b || !bm_reserve(b, ix->size)) { *error = "Out of memory!"; goto fail; }
    for (uint32_t s = 0; s < ix->size; ++s) {
        int16_t const level = rd_i16((uint8_t const*)ix->levels + 2u * s);
        b->levels[s] = level;
        b->linked_in[s] = b->written_in[s] = -1;
        b->keys[s] = node_key(ix, s);
        memcpy(b->vectors + (size_t)s * b->bytes_per_vector, ix->vectors + (size_t)s * ix->bytes_per_vector, b->bytes_per_vector);
        if (!bm_alloc_rows(b, s, level)) { *error = "Out of memory!"; b->size = s; goto fail; }
        b->size = s + 1;
        for (int l = 0; l <= level; ++l) {
            uint8_t const* nb = l ? neighbors_non_base(ix, s, (size_t)l) : neighbors_base(ix, s);
            uint32_t const n = rd_u32(nb);
            if (n > bm_capacity_of(b, (size_t)l)) { *error = "List longer than its level's capacity"; goto fail; }
            for (uint32_t i = 0; i < n; ++i) bm_row(b, s, (size_t)l)[i] = rd_u32(nb + 4 + 4 * i);
        }
    }
    b->linked = b->size;
    b->entry = (uint32_t)ix->entry_slot;
    b->max_level = (int)ix->max_level;
    f64 ? oracle_close_f64(ix) : oracle_close(ix);
    return b;
fail:
    f64 ? oracle_close_f64(ix) : oracle_close(ix);
    bm_free(b);
    return NULL;
}

/* ---- the INSERT search of one task ------------------------------------------------------------------------------- */

/* search_for_one_ over the model's rows: greedy descent from `closest` on begin_level down to end_level + 1 */
static uint32_t bm_descend(bm_index_t* b, void const* q, uint32_t closest, int begin_level, int end_level) {
    float closest_dist = bm_measure(b, q, closest);
    for (int level = begin_level; level > end_level; --level) {
        int changed;
        do {
            changed = 0;
            uint32_t const* row = bm_row(b, closest, (size_t)level); /* the list of the node held at loop entry */
            size_t const n = bm_listed(b, closest, (size_t)level);
            for (size_t i = 0; i < n; ++i) {
                float const d = bm_measure(b, q, row[i]);
                if (d < closest_dist) { closest_dist = d; closest = row[i]; changed = 1; }
            }
        } while (changed);
    }
    return closest;
}

/* search_to_insert_ on `level` from `start`, ef = top_limit; `self` (a reused member's slot) never enters `top`.
 * Leaves the candidates, ascending, in b->ctx.top. */
static int bm_search_level(bm_index_t* b, void const* q, uint32_t self, uint32_t start, size_t level, size_t top_limit) {
    context_t* c = &b->ctx;
    heap_t* next = &c->next;
    sorted_t* top = &c->top;
    visits_t* visits = &c->visits;
    visits_clear(visits);
    next->size = 0;
    top->size = 0;
    if (!visits_reserve(visits, b->m0 + 1u) || !heap_reserve(next, top_limit)) return 0;
    if (top->capacity < top_limit + 1) {
        candidate_t* e = (candidate_t*)realloc(top->e, (top_limit + 1) * sizeof(candidate_t));
        if (!e) return 0;
        top->e = e;
        top->capacity = top_limit + 1;
    }
    float radius = bm_measure(b, q, start);
    candidate_t seed = {-radius, start};
    next->e[next->size++] = seed;
    visits_set(visits, start);
    if (start != self) {
        candidate_t t = {radius, start};
        sorted_insert_reserved(top, t);
    }
    while (next->size) {
        candidate_t cand = next->e[0];
        if ((-cand.distance) > radius && top->size == top_limit) break;
        heap_pop(next);
        c->iteration_cycles++;
        uint32_t const* row = bm_row(b, cand.slot, level);
        size_t const n = bm_listed(b, cand.slot, level);
        if (!visits_reserve(visits, visits->count + n)) return 0;
        for (size_t i = 0; i < n; ++i) {
            uint32_t const succ = row[i];
            if (visits_set(visits, succ)) continue;
            float const d = bm_measure(b, q, succ);
            if (top->size < top_limit || d < radius) {
                candidate_t neg = {-d, succ};
                if (!heap_insert(next, neg)) return 0;
                if (succ != self) {
                    candidate_t pos = {d, succ};
                    sorted_insert(top, pos, top_limit);
                    radius = top->e[top->size - 1].distance;
                }
            }
        }
    }
    return 1;
}

/* the candidates of one task as the INSERT kernel returns them: descent to level + 1, then the level's search */
static int bm_task_search(bm_index_t* b, void const* q, uint32_t self, size_t level, size_t ef) {
    uint32_t const closest = bm_descend(b, q, b->entry, b->max_level, (int)level);
    return bm_search_level(b, q, self, closest, level, ef);
}

/* exported for the tests: candidates of a query row on `level` over the current graph (self = EMPTY_SLOT: none) */
long bm_candidates(bm_index_t* b, void const* query, uint32_t self, size_t level, size_t ef, uint32_t* slots, float* dists) {
    if (!b->linked) return 0;
    if (!bm_task_search(b, query, self, level, ef)) return -1;
    for (size_t i = 0; i < b->ctx.top.size; ++i) {
        slots[i] = b->ctx.top.e[i].slot;
        dists[i] = b->ctx.top.e[i].distance;
    }
    return (long)b->ctx.top.size;
}

/* ---- refine_ --------------------------------------------------------------------------------------------------- */

/* `cand` ascending by distance to the centre; keeps the first, then candidate c iff no kept s has d(c, s) < d(c, centre),
 * at most `needed`. With fewer candidates than needed all are kept (in the order given). Returns the number kept,
 * compacted at the front of `cand`. */
static size_t bm_refine(bm_index_t* b, candidate_t* cand, size_t count, size_t needed) {
    if (count < needed) return count;
    size_t kept = 1;
    for (size_t c = 1; c < count && kept < needed; ++c) {
        int good = 1;
        for (size_t s = 0; s < kept && good; ++s)
            if (b->metric(bm_vec(b, cand[c].slot), bm_vec(b, cand[s].slot), b->third) < cand[c].distance) good = 0;
        if (good) cand[kept++] = cand[c];
    }
    return kept;
}

/* ---- one batch ------------------------------------------------------------------------------------------------- */

typedef struct { uint64_t key; uint32_t index; uint32_t member; float distance; } bm_pair_t;

static int bm_pair_order(void const* x, void const* y) {
    bm_pair_t const* a = (bm_pair_t const*)x;
    bm_pair_t const* b = (bm_pair_t const*)y;
    if (a->key != b->key) return a->key < b->key ? -1 : 1;
    return a->index < b->index ? -1 : a->index > b->index;
}

static int bm_candidate_order(void const* x, void const* y) { /* ascending distance, NaN after every number, ties by slot */
    candidate_t const* a = (candidate_t const*)x;
    candidate_t const* b = (candidate_t const*)y;
    int const na = a->distance != a->distance, nb = b->distance != b->distance;
    if (na != nb) return na ? 1 : -1;
    if (!na && a->distance != b->distance) return a->distance < b->distance ? -1 : 1;
    return a->slot < b->slot ? -1 : a->slot > b->slot;
}

static int bm_link_batch(bm_index_t* b, uint32_t const* slots, size_t count, size_t ef) {
    int const top_level = b->max_level;
    int32_t const batch = (int32_t)b->counters[BM_BATCHES];
    size_t ntasks = count;
    for (size_t i = 0; i < count; ++i) ntasks += (size_t)(b->levels[slots[i]] < top_level ? b->levels[slots[i]] : top_level);
    uint32_t* t_slot = (uint32_t*)malloc(ntasks * 4 + 4);
    uint8_t* t_level = (uint8_t*)malloc(ntasks + 1);
    candidate_t* cands = (candidate_t*)malloc(ntasks * BM_CAND_MAX * sizeof(candidate_t) + 1);
    size_t* ncands = (size_t*)malloc(ntasks * sizeof(size_t) + 1);
    bm_pair_t* pairs = (bm_pair_t*)malloc(ntasks * b->m * sizeof(bm_pair_t) + 1);
    int ok = t_slot && t_level && cands && ncands && pairs;
    size_t t = 0, npairs = 0;
    if (!ok) goto done;
    for (size_t i = 0; i < count; ++i) { t_slot[t] = slots[i]; t_level[t++] = 0; }
    for (size_t i = 0; i < count; ++i)
        for (int l = 1; l <= b->levels[slots[i]] && l <= top_level; ++l) { t_slot[t] = slots[i]; t_level[t++] = (uint8_t)l; }

    /* 1. candidates, all over the graph as it stands before the batch */
    for (t = 0; t < ntasks && ok; ++t) {
        ok = bm_task_search(b, bm_vec(b, t_slot[t]), t_slot[t], t_level[t], ef);
        size_t n = b->ctx.top.size < ef ? b->ctx.top.size : ef;
        if (n > BM_CAND_MAX) { n = BM_CAND_MAX; b->counters[BM_CANDIDATE_CUTS]++; }
        memcpy(cands + t * BM_CAND_MAX, b->ctx.top.e, n * sizeof(candidate_t));
        ncands[t] = n;
    }
    if (!ok) goto done;
    /* 2. forward: each task writes its member's row on its level and emits its pairs */
    for (t = 0; t < ntasks; ++t) {
        candidate_t* c = cands + t * BM_CAND_MAX;
        if (ncands[t] < b->m) b->counters[BM_SHORT_REFINES]++;
        size_t const kept = bm_refine(b, c, ncands[t], b->m);
        uint32_t* row = bm_row(b, t_slot[t], t_level[t]);
        for (size_t i = 0; i < bm_capacity_of(b, t_level[t]); ++i) row[i] = i < kept ? c[i].slot : BM_EMPTY;
        b->linked_in[t_slot[t]] = b->written_in[t_slot[t]] = batch;
        for (size_t i = 0; i < kept; ++i) {
            bm_pair_t const p = {((uint64_t)t_level[t] << 32) | c[i].slot, (uint32_t)(t * b->m + i), t_slot[t], c[i].distance};
            pairs[npairs++] = p;
        }
    }
    /* 3. pairs grouped by (level, neighbour), index order inside a group */
    qsort(pairs, npairs, sizeof(bm_pair_t), bm_pair_order);
    /* 4. reverse: one run per (level, neighbour); each writes only its own row */
    for (size_t p0 = 0; p0 < npairs;) {
        size_t p1 = p0;
        while (p1 < npairs && pairs[p1].key == pairs[p0].key) ++p1;
        b->counters[BM_REVERSE_RUNS]++;
        size_t const level = (size_t)(pairs[p0].key >> 32);
        uint32_t const centre = (uint32_t)pairs[p0].key;
        uint32_t* row = bm_row(b, centre, level);
        size_t const capacity = bm_capacity_of(b, level);
        size_t const listed = bm_listed(b, centre, level);
        size_t const room = BM_CAND_MAX - (listed < BM_CAND_MAX ? listed : BM_CAND_MAX);
        size_t run = p1 - p0;
        if (run > room) { run = room; b->counters[BM_ROOM_CUTS]++; }
        b->written_in[centre] = batch;
        candidate_t all[BM_CAND_MAX];
        size_t arrivals = 0;
        for (size_t i = 0; i < run; ++i) {
            uint32_t const s = pairs[p0 + i].member;
            int held = 0;
            for (size_t j = 0; j < listed && !held; ++j) held = row[j] == s;
            if (held) { b->counters[BM_HELD_ARRIVALS]++; continue; }
            all[listed + arrivals].slot = s;
            all[listed + arrivals].distance = pairs[p0 + i].distance;
            ++arrivals;
        }
        if (listed + arrivals <= capacity) {
            for (size_t i = 0; i < arrivals; ++i) row[listed + i] = all[listed + i].slot;
        } else {
            b->counters[BM_REVERSE_REFINES]++;
            if (!level) b->counters[BM_REVERSE_REFINES_BASE]++;
            for (size_t i = 0; i < listed; ++i) {
                all[i].slot = row[i];
                all[i].distance = b->metric(bm_vec(b, centre), bm_vec(b, row[i]), b->third);
            }
            qsort(all, listed + arrivals, sizeof(candidate_t), bm_candidate_order);
            for (size_t i = 1; i < listed + arrivals; ++i)
                if (all[i].distance == all[i - 1].distance) { b->counters[BM_SORT_TIES]++; break; }
            size_t const kept = bm_refine(b, all, listed + arrivals, capacity);
            for (size_t i = 0; i < capacity; ++i) row[i] = i < kept ? all[i].slot : BM_EMPTY;
        }
        p0 = p1;
    }
    /* after the batch: the entry point and the top level */
    for (size_t i = 0; i < count; ++i) {
        if (b->levels[slots[i]] > b->max_level) { b->max_level = b->levels[slots[i]]; b->entry = slots[i]; }
        if ((size_t)slots[i] + 1 > b->linked) b->linked = (size_t)slots[i] + 1;
    }
    b->counters[BM_BATCHES]++;
    b->counters[BM_TASKS] += ntasks;
done:
    free(t_slot);
    free(t_level);
    free(cands);
    free(ncands);
    free(pairs);
    return ok;
}

static size_t bm_min3(size_t a, size_t b, size_t c) { size_t m = a < b ? a : b; return m < c ? m : c; }

/* `count` rows (stored scalar kind, `stride` bytes apart) under `keys`: the first min(count, nreuse) go into the slots of
 * `reuse` in order and keep those slots' levels, the rest are appended with levels `levels[0..)`. Returns 0 on success. */
int bm_add(bm_index_t* b, uint64_t const* keys, void const* rows, size_t count, size_t stride, int16_t const* levels,
           uint32_t const* reuse, size_t nreuse, size_t expansion_add, size_t batch_cap, size_t ratio) {
    if (!count) return 0;
    size_t const reused = count < nreuse ? count : nreuse;
    size_t const appended = count - reused;
    size_t const first = b->size;
    size_t const ef = expansion_add ? expansion_add : 128;
    if (!batch_cap) batch_cap = 32768;
    if (!ratio) ratio = 32;
    if (!bm_reserve(b, first + appended)) return -1;
    uint8_t const* src = (uint8_t const*)rows;
    for (size_t i = 0; i < reused; ++i) {
        if (reuse[i] >= b->linked) return -2;
        memcpy(b->vectors + (size_t)reuse[i] * b->bytes_per_vector, src + i * stride, b->bytes_per_vector);
        b->keys[reuse[i]] = keys[i];
    }
    for (size_t i = 0; i < appended; ++i) {
        uint32_t const s = (uint32_t)(first + i);
        memcpy(b->vectors + (size_t)s * b->bytes_per_vector, src + (reused + i) * stride, b->bytes_per_vector);
        b->keys[s] = keys[reused + i];
        b->levels[s] = levels[i];
        b->linked_in[s] = b->written_in[s] = -1;
        if (!bm_alloc_rows(b, s, levels[i])) return -1;
        b->size = s + 1;
    }
    /* reused members keep their level (<= the top level): their batches are never cut */
    for (size_t at = 0; at < reused;) {
        size_t const batch = bm_min3(reused - at, batch_cap, b->linked / ratio > 1 ? b->linked / ratio : 1);
        if (!bm_link_batch(b, reuse + at, batch, ef)) return -1;
        b->counters[BM_REUSED] += batch;
        at += batch;
    }
    uint32_t* batch_slots = (uint32_t*)malloc((batch_cap < appended ? batch_cap : appended) * 4 + 4);
    if (!batch_slots) return -1;
    for (size_t at = first; at < b->size;) {
        if (b->linked == 0) { /* the first member: entry point, no links */
            b->entry = (uint32_t)at;
            b->max_level = b->levels[at];
            b->linked = 1;
            at += 1;
            continue;
        }
        size_t batch = bm_min3(b->size - at, batch_cap, b->linked / ratio > 1 ? b->linked / ratio : 1);
        for (size_t i = 0; i < batch; ++i)
            if (b->levels[at + i] > b->max_level) { batch = i + 1; break; }
        for (size_t i = 0; i < batch; ++i) batch_slots[i] = (uint32_t)(at + i);
        if (!bm_link_batch(b, batch_slots, batch, ef)) { free(batch_slots); return -1; }
        at += batch;
    }
    free(batch_slots);
    return 0;
}

/* ---- read-out ---------------------------------------------------------------------------------------------------- */

size_t bm_size(bm_index_t const* b) { return b->size; }
size_t bm_connectivity(bm_index_t const* b) { return b->m; }
size_t bm_connectivity_base(bm_index_t const* b) { return b->m0; }
size_t bm_entry(bm_index_t const* b) { return b->entry; }
long bm_max_level(bm_index_t const* b) { return b->max_level; }
size_t bm_upper_rows(bm_index_t const* b) {
    size_t rows = 0;
    for (size_t i = 0; i < b->size; ++i) rows += (size_t)b->levels[i];
    return rows;
}

/* levels [size], keys [size], level-0 rows [size x m0], upper rows [upper_rows x m] in slot order then level order */
void bm_export(bm_index_t const* b, int16_t* levels, uint64_t* keys, uint32_t* rows0, uint32_t* upper) {
    size_t u = 0;
    for (size_t s = 0; s < b->size; ++s) {
        levels[s] = b->levels[s];
        keys[s] = b->keys[s];
        memcpy(rows0 + s * b->m0, b->rows[s], b->m0 * 4);
        memcpy(upper + u * b->m, b->rows[s] + b->m0, (size_t)b->levels[s] * b->m * 4);
        u += (size_t)b->levels[s];
    }
}

void bm_batches(bm_index_t const* b, int32_t* linked_in, int32_t* written_in) {
    memcpy(linked_in, b->linked_in, b->size * 4);
    memcpy(written_in, b->written_in, b->size * 4);
}
void bm_vectors(bm_index_t const* b, uint8_t* out) { memcpy(out, b->vectors, b->size * b->bytes_per_vector); }
void bm_counters(bm_index_t const* b, uint64_t* out) { memcpy(out, b->counters, sizeof(b->counters)); }
float bm_distance(bm_index_t const* b, uint32_t a, uint32_t c) { return b->metric(bm_vec(b, a), bm_vec(b, c), b->third); }
