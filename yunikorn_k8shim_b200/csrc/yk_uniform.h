// yk_uniform.h -- the device-resident ordered commit for a UNIFORM RUN: a stretch of consecutive asks in the orderer's
// order that all request the same vector and carry the same predicate signature (the replicas of one deployment / the
// executors of one job; the reference's own benchmark, pkg/shim/scheduler_perf_test.go:283-288, is one such run of 50 000).
// Single source like yk_lattice.h: the per-item bodies below are called by the sm_90a kernels in yk_uniform.cuh and, as
// plain loops, by tests/host/lattice_shim.cpp (test infrastructure).
//
// What it replaces: the same one-allocation-per-pass loop as yk_lattice.h [EXT yunikorn-core Application.tryNodes, entered
// per pair through pkg/cache/scheduler_callback.go:196-198 -> pkg/cache/context.go:683-703], under the `fair` node sort.
//
// Why a uniform run has no sequential part at all.  Under `fair` a node's key never decreases when it is allocated to
// (yk_lattice_host.hpp eligible()).  Node n can take the request cap_n more times; its j-th allocation of the run happens
// while the node is in state j, whose key k_n(j) = score(available - j * request) is known in advance and monotone in j.
// The sequential loop "minimum (key, NodeID) over the nodes that pass; allocate; re-key" therefore takes the ELEMENTS
// (n, j), j < cap_n, in ascending (k_n(j), NodeID rank, j) order: ask i of the run gets the node of the i-th element.
// That is one stable radix sort of the element keys (elements generated in (rank, j) order) and a gather -- grid-wide,
// no chain.  Elements are generated to a depth L per node; the selection is exact iff the last element taken sorts
// before the first element NOT generated (the smallest (k_n(L), rank_n) over the nodes cut at L): checked on the device,
// a violation asks the host for a deeper L and nothing is applied.
#pragma once
#include <stdint.h>
#include "yk_lattice.h"

namespace ykun {

constexpr uint64_t KEY_INF = yklt::KEY_INF;   // = YK_KEY_NAN: a generated element with this key is a NaN score
constexpr uint32_t NONE = yklt::NONE;

enum { U_DONE = 0, U_STOPPED = 1, U_RETRY = 2, U_FALLBACK = 3, U_NAN = 4 };

// grid-wide scalars of one attempt
struct Globals {
    unsigned long long bkey;        // smallest key of a first not-generated element (KEY_INF: no node was cut at L)
    unsigned long long brank;       // ... and the smallest rank among the nodes that have it
    unsigned long long last_key;    // the last element taken
    unsigned long long last_rank;
    unsigned int valid;             // generated elements
    int nan;
    int status;
    int consumed;                   // entries of the run decided
};

struct Args {
    uint32_t policy;
    double w[8];
    int64_t* rec; int RS;            // node records (yk_lattice.h Args::rec)
    yklt::Ent* ord[2]; const int* cur;
    int nlive;
    const uint32_t* byrank;          // [nlive] the live nodes in ascending NodeID rank
    int64_t req[8];                  // the run's request
    uint64_t tol, need, deny; uint32_t want;   // ... and predicate signature
    int L;                           // elements generated per node
    int R;                           // asks in the run
    int insensitive, has_gang;
    unsigned long long* ekey; uint32_t* enode;         // [nlive * L] generated, (rank, j) order (binpacking fill, once sorted:
                                                       // the capacity per sorted position)
    const unsigned long long* skey; const uint32_t* snode;   // the same, stably sorted by key
    unsigned long long* bk;          // [nlive] key of element (n, L) where the node was cut, else KEY_INF (binpacking fill, once
                                     // sorted: the inclusive sum of the capacities)
    uint32_t* cnt;                   // [node index] elements taken per node; zero outside an attempt
    unsigned long long* rkey; unsigned long long* rrn;           // [nlive] re-keyed order entries in rank order
    const unsigned long long* okey; const unsigned long long* orn;   // ... sorted by key
    uint32_t* res;                   // [R] node index or NONE
    Globals* g;
};

// how many more times `req` fits the node (yklt::fits applied repeatedly), at most `limit`
template <int D>
LT_HD int64_t cap_of(bool usable, const int64_t* avail, const int64_t* total, const int64_t* req, int64_t limit) {
    if (!usable) return 0;
    int64_t c = limit;
    for (int k = 0; k < D; ++k) {
        const int64_t r = req[k];
        if (r <= 0) continue;   // r <= max(0, .) always holds
        const int64_t t = total[k] < 0 ? 0 : total[k];
        const int64_t a = avail[k] < 0 ? 0 : avail[k];
        if (r > t) return 0;
        const int64_t q = a / r;
        c = q < c ? q : c;
    }
    return c;
}

// the same with the dimension count at run time (host side)
inline int64_t cap_of_d(int D, bool usable, const int64_t* avail, const int64_t* total, const int64_t* req, int64_t limit) {
    if (!usable) return 0;
    int64_t c = limit;
    for (int k = 0; k < D; ++k) {
        const int64_t r = req[k];
        if (r <= 0) continue;
        const int64_t t = total[k] < 0 ? 0 : total[k];
        const int64_t a = avail[k] < 0 ? 0 : avail[k];
        if (r > t) return 0;
        const int64_t q = a / r;
        c = q < c ? q : c;
    }
    return c;
}

struct DepthOut { unsigned int valid; unsigned long long bk; int nan; };

// element x = i * L + j: state j of node i (rank order).  The thread of j = 0 also reports the node's depth and, where the
// node was cut at L, the key of its first element that is not generated.
template <int D>
LT_FN DepthOut element_item(const Args& a, long long x) {
    const int L = a.L;
    const int i = (int)(x / L), j = (int)(x % L);
    const uint32_t n = a.byrank[i];
    const int64_t* r = a.rec + (size_t)n * a.RS;
    const uint32_t fl = (uint32_t)(uint64_t)r[2 * D + 2];
    const bool usable = (fl & 1u) && !(fl & 2u);
    const bool acc = yklt::accepts((uint64_t)r[2 * D], (uint64_t)r[2 * D + 1], n, a.tol, a.need, a.deny, a.want);
    const int64_t cap = acc ? cap_of<D>(usable, r, r + D, a.req, (int64_t)a.R) : 0;
    DepthOut o; o.valid = 0; o.bk = KEY_INF; o.nan = 0;
    int64_t av[D];
    unsigned long long key = KEY_INF;
    if ((int64_t)j < cap) {
        for (int k = 0; k < D; ++k) av[k] = r[k] - (int64_t)j * a.req[k];
        key = yklt::key_of<D>(a.policy, a.w, r + D, av);
        if (key == KEY_INF) o.nan = 1;
    }
    a.ekey[x] = key; a.enode[x] = n;
    if (j == 0) {
        o.valid = (unsigned)(cap < (int64_t)L ? cap : (int64_t)L);
        if (cap > (int64_t)L) {
            for (int k = 0; k < D; ++k) av[k] = r[k] - (int64_t)L * a.req[k];
            o.bk = yklt::key_of<D>(a.policy, a.w, r + D, av);   // state L
            if (o.bk == KEY_INF) o.nan = 1;
        }
        a.bk[i] = o.bk;
    }
    return o;
}

// rank of node i if it holds the smallest cut key, else KEY_INF
template <int D>
LT_FN unsigned long long brank_item(const Args& a, int i, unsigned long long bkey) {
    if (bkey == KEY_INF || a.bk[i] != bkey) return KEY_INF;
    const uint32_t n = a.byrank[i];
    return (unsigned long long)((uint64_t)a.rec[(size_t)n * a.RS + 2 * D + 2] >> 32);
}

// what the attempt amounts to (one thread, after the selection)
LT_FN void decide(const Args& a) {
    Globals& g = *a.g;
    const unsigned m = g.valid < (unsigned)a.R ? g.valid : (unsigned)a.R;
    const bool cut = g.bkey != KEY_INF;
    if (g.nan) { g.status = U_NAN; g.consumed = 0; return; }
    if (cut) {
        // exact iff everything taken sorts before the first element that was not generated.  Ranks are unique, so an equal
        // (key, rank) is the cut node itself: its generated states come first (j < L).
        const bool ok = m == (unsigned)a.R && (g.last_key < g.bkey || (g.last_key == g.bkey && g.last_rank <= g.brank));
        if (!ok) { g.status = U_RETRY; g.consumed = 0; return; }
    }
    if (m < (unsigned)a.R) {
        // every element there is was generated: asks m, m+1, ... find nothing
        if (a.has_gang) { g.status = U_FALLBACK; g.consumed = 0; return; }   // a gang may have to be rolled back: the windowed commit does that
        if (a.insensitive) { g.status = U_DONE; g.consumed = a.R; return; }
        g.status = U_STOPPED; g.consumed = (int)m + 1;
        return;
    }
    g.status = U_DONE; g.consumed = a.R;
}

// ask q of the run: the node of the q-th element
template <int D>
LT_FN void select_item(const Args& a, int q, unsigned valid) {
    const unsigned m = valid < (unsigned)a.R ? valid : (unsigned)a.R;
    if ((unsigned)q >= m) { a.res[q] = NONE; return; }
    const uint32_t n = a.snode[q];
    a.res[q] = n;
#if defined(__CUDA_ARCH__)
    atomicAdd(&a.cnt[n], 1u);
#else
    a.cnt[n] += 1u;
#endif
    if ((unsigned)q == m - 1) {
        a.g->last_key = a.skey[q];
        a.g->last_rank = (unsigned long long)((uint64_t)a.rec[(size_t)n * a.RS + 2 * D + 2] >> 32);
    }
}

// node i: available -= taken * request (when the attempt stands); the counter is cleared either way
template <int D>
LT_FN void apply_item(const Args& a, int i, int status) {
    const uint32_t n = a.byrank[i];
    const uint32_t c = a.cnt[n];
    if (c == 0) return;
    a.cnt[n] = 0;
    if (status != U_DONE && status != U_STOPPED) return;
    int64_t* r = a.rec + (size_t)n * a.RS;
    for (int k = 0; k < D; ++k) r[k] -= (int64_t)c * a.req[k];
}

// node i: its order entry under the current availability
template <int D>
LT_FN int rekey_item(const Args& a, int i) {
    const uint32_t n = a.byrank[i];
    const int64_t* r = a.rec + (size_t)n * a.RS;
    const unsigned long long key = yklt::key_of<D>(a.policy, a.w, r + D, r);
    a.rkey[i] = key;
    a.rrn[i] = ((uint64_t)r[2 * D + 2] >> 32 << 32) | (uint64_t)n;
    return key == KEY_INF ? 1 : 0;
}

// ---- binpacking: one ordered capacity fill per run (DESIGN.md §6.4) ----------------------------------------------------
// Under `binpacking` (key = 1 - usage) a node's key never INCREASES when it is allocated to.  So the node at the front of the
// ascending (key, rank) order among those that accept the run and have room keeps taking its asks until its capacity for the
// request is gone; a node before it refused the run by its masks or flags or had no room, and neither changes during the
// run.  Ask q of the run therefore goes to the node where the inclusive prefix sum of the capacities, in that order, first
// exceeds q: element_item at L = 1 gives the keys (KEY_INF where the node takes nothing), a stable radix sort of them in
// rank order gives skey / snode, then fill_cap_item (into ekey), a 64-bit inclusive scan of ekey into bk (nodes x R
// overflows 32 bits), fill_decide, fill_select_item and the unchanged apply / re-key.  No depth, no retry, no chain.

// sorted position p: how many asks of the run its node takes (at most R; 0 past the nodes that take any)
template <int D>
LT_FN void fill_cap_item(const Args& a, int p) {
    if (a.skey[p] == KEY_INF) { a.ekey[p] = 0; return; }
    const int64_t* r = a.rec + (size_t)a.snode[p] * a.RS;
    a.ekey[p] = (unsigned long long)cap_of<D>(true, r, r + D, a.req, (int64_t)a.R);   // a finite key: usable, accepts, cap >= 1
}

// what the fill amounts to (one thread, after the scan): decide() without RETRY; g.valid = the asks that get a node
LT_FN void fill_decide(const Args& a) {
    Globals& g = *a.g;
    const unsigned long long total = a.nlive > 0 ? a.bk[a.nlive - 1] : 0ull;
    const unsigned m = total < (unsigned long long)a.R ? (unsigned)total : (unsigned)a.R;
    g.valid = m;
    if (g.nan) { g.status = U_NAN; g.consumed = 0; return; }
    if (m < (unsigned)a.R) {   // asks m, m+1, ... find nothing
        if (a.has_gang) { g.status = U_FALLBACK; g.consumed = 0; return; }   // a gang may have to be rolled back: the host commit does that
        if (a.insensitive) { g.status = U_DONE; g.consumed = a.R; return; }
        g.status = U_STOPPED; g.consumed = (int)m + 1;
        return;
    }
    g.status = U_DONE; g.consumed = a.R;
}

// ask q of the run (select_item's contract): the node of the first sorted position whose inclusive sum exceeds q
LT_FN void fill_select_item(const Args& a, int q, unsigned m) {
    if ((unsigned)q >= m) { a.res[q] = NONE; return; }
    int lo = 0, hi = a.nlive - 1;   // bk[nlive - 1] >= m > q
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a.bk[mid] > (unsigned long long)q) hi = mid; else lo = mid + 1;
    }
    const uint32_t n = a.snode[lo];
    a.res[q] = n;
#if defined(__CUDA_ARCH__)
    atomicAdd(&a.cnt[n], 1u);
#else
    a.cnt[n] += 1u;
#endif
}

// ---- host side: where the uniform runs of a batch are ------------------------------------------------------------
struct Segment { int off, len; bool uniform; };

// Cuts [0, B) into uniform runs of at least min_run entries and the stretches between them.  A run never starts or ends
// inside a gang (gang members carry M_GANG, the first one M_GSTART).
template <typename Vec>
inline void plan_segments(const uint32_t* meta, const uint32_t* shp, const uint32_t* sig, int B, int min_run, Vec& out) {
    out.clear();
    int open = 0;   // start of the stretch not yet emitted
    int i = 0;
    while (i < B) {
        int j = i + 1;
        while (j < B && shp[j] == shp[i] && sig[j] == sig[i]) ++j;
        int s = i, e = j;
        auto inside_gang = [&](int x) { return x < B && (meta[x] & yklt::M_GANG) && !(meta[x] & yklt::M_GSTART); };
        while (s < e && inside_gang(s)) ++s;
        while (e > s && inside_gang(e)) --e;
        if (e - s >= min_run) {
            if (s > open) out.push_back(Segment{open, s - open, false});
            out.push_back(Segment{s, e - s, true});
            open = e;
        }
        i = j;
    }
    if (open < B) out.push_back(Segment{open, B - open, false});
}

// first depth to try: twice the mean share of a node, a power of two
inline int first_depth(int R, int nlive) {
    const long long mean = nlive > 0 ? ((long long)R + nlive - 1) / nlive : 1;
    int L = 4;
    while (L < 2 * mean + 2 && L < (1 << 20)) L <<= 1;
    return L;
}

}  // namespace ykun
