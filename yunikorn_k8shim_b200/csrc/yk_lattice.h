// yk_lattice.h -- the device-resident ordered commit ("lattice commit"), single source:
//   * compiled by nvcc it is the body of yk_lattice_kernel (one persistent CTA of 1024 threads, sm_90a);
//   * compiled by g++ (tests/host/device_shim.cpp) the SAME code runs as a sequential emulation, so the CPU test suite
//     fuzzes the algorithm against the oracle without a GPU (test infrastructure; the product only ever runs the kernel).
//
// What it replaces: the reference's one-allocation-per-pass loop [EXT yunikorn-core Application.tryNodes / tryNode, entered
// per (ask,node) pair through pkg/cache/scheduler_callback.go:196-198 -> pkg/cache/context.go:683-703 ->
// pkg/plugin/predicates/predicate_manager.go:130-283] under the `fair` node-sort policy, for a WINDOW of consecutive asks
// that request at most SMAX distinct resource vectors ("shapes": the replicas of a few deployments / jobs / task groups).
//
// Why a window is parallel.  Under `fair` a node's key (float64 usage score, SURVEY A.3) never decreases when something is
// allocated on it.  Within a window a node is in a STATE c = (c_1..c_S): how many allocations of each shape it has taken.
// State c of node n has a key k_n(c) that is known in advance (available - sum c_s r_s, re-scored), and k_n is monotone in
// every c_s.  The sequential loop "take the minimum (key, NodeID) over the nodes that pass, allocate, re-key" therefore
// walks a LATTICE of elements (node, state): an ask of shape s takes the first element, in (key, NodeID) order, that is
// currently AVAILABLE (its node is in exactly that state), has room for one more s, and whose node passes the ask's own
// taint / affinity / node-name masks; the element becomes unavailable and its child (node, c + e_s) becomes available.
// All of that is bit arithmetic on a sorted element list:   first set bit of  AVAIL & ROOM_s & ACCEPT_sig   per ask --
// a few register operations for one warp -- while everything else (which states exist, their float64 keys, the room and
// mask tests, the child links, the new node order) is evaluated in parallel by the whole CTA.
//
// One sub-run =
//   1. stage   the next asks up to SMAX distinct shapes / SIGCAP distinct signatures; never cut inside a gang
//   2. scan    the first P positions of the node order (ascending (key, NodeID)), gather their records
//   3. window  choose a key threshold tau (largest of eight candidates whose state count fits) and per node / shape the
//              depth d_s = how many allocations of s alone stay below tau; the node's states are the box [0,d_1]x..x[0,d_S]
//   4. bound   the smallest key just outside any box ((d_s+1) e_s: boxes are cut along the axes and keys are monotone)
//              and the key of position P: every element below the bound is known, so the sorted list below it is exact
//   5. lattice evaluate the box states (reachable? key below the bound?), sort when there is more than the bases
//   6. links   child of (element, shape), ROOM_s bitmaps, one ACCEPT bitmap per distinct predicate signature
//   7. chain   warp 0, sequential over the asks; gangs snapshot / restore the AVAIL words
//   8. apply   available -= sum c_s r_s on the touched nodes, float64 re-score, bindings out
//   9. patch   the touched nodes leave their positions and are merged back by their new keys
// An ask that finds nothing below the bound ends the sub-run there (the next one starts from the new order); an ask that
// finds nothing in a fresh sub-run is decided by a full scan of the order (exact first fit, or certain NOFIT, which also
// refreshes the per-dimension capacity bound that rejects later hopeless asks without a scan).
#pragma once
#include <stdint.h>
#include "yk_score.h"

#ifndef YK_LT_THREADS
#define YK_LT_THREADS 1024
#endif

#if defined(__CUDACC__)
#define LT_DEV 1
#define LT_HD __host__ __device__ __forceinline__
#define LT_FN __device__ __forceinline__
#define LT_NI __device__ __noinline__   /* the phases run once per sub-run: code size (instruction fetch), not call overhead, is what costs */
#define LT_FOR(i, n) _Pragma("unroll 1") for (int i = (int)threadIdx.x; i < (int)(n); i += yklt::THREADS)
#define LT_FOR32(i, n) _Pragma("unroll 1") for (int i = (int)threadIdx.x; i < (((int)(n) + 31) & ~31); i += yklt::THREADS)   /* whole warps */
#define LT_SYNC() __syncthreads()
#define LT_ONE if (threadIdx.x == 0)
#define LT_PROF(k) do { if (a.prof && threadIdx.x == 0) { const long long _t = clock64(); a.prof[k] += _t - prof_t; prof_t = _t; } } while (0)
#else
#define LT_DEV 0
#define LT_HD inline
#define LT_FN inline
#define LT_NI inline
#define LT_FOR(i, n) for (int i = 0; i < (int)(n); ++i)
#define LT_FOR32(i, n) for (int i = 0; i < (int)(n); ++i)
#define LT_SYNC() ((void)0)
#define LT_ONE if (true)
#define LT_PROF(k) ((void)0)
#endif

namespace yklt {

constexpr int THREADS = YK_LT_THREADS;
constexpr int LCAP = 2048;              // lattice elements of one sub-run
constexpr int FW = LCAP / 32;           // words per bitmap over the elements
constexpr int KCAP = 512;               // asks per sub-run
constexpr int SIGCAP = 128;             // distinct predicate signatures per sub-run
constexpr int SMAX = 8;                 // distinct request vectors ("shapes") per sub-run
constexpr int DCAP = 63;                // deepest a box goes along one shape
constexpr int VCAP = 256;               // states per node
constexpr int HT = 1024;                // slots of the per-sub-run id tables (shape ids, signature ids)
constexpr int NCAND = 6;                // candidate key thresholds per sub-run
constexpr int ECNT = 512;               // up to this many non-base elements are merged in by counting, more by a bitonic sort
constexpr uint32_t NONE = 0xFFFFFFFFu;
constexpr uint16_t NO_CHILD = 0xFFFFu;
constexpr uint64_t KEY_INF = 0xFFFFFFFFFFFFFFFFull;

// Per batch entry the host (which knows requests, signatures and gangs) writes three words:
//   meta  flags;  shp  a number that is equal exactly for equal request vectors;  sig  a number that is equal exactly for
//   equal predicate signatures (request, tolerations, required / forbidden labels, node name)
constexpr uint32_t M_GSTART = 4;        // first member of a gang
constexpr uint32_t M_GANG = 8;          // member of a gang

// hdr[] words
enum { H_CONSUMED = 0, H_STATUS = 1, H_SUBRUNS = 2, H_FULLSCANS = 3, H_SORTS = 4, H_ELEMS = 5, H_QUICK = 6, H_ESC = 7, H_WORDS = 8 };
enum { ST_DONE = 0, ST_STOPPED = 1, ST_HANDOFF = 2, ST_NAN = 3 };

struct Ent { uint64_t key; uint64_t rn; };   // one position of the node order: sort key, NodeID rank << 32 | node index

LT_HD bool ent_less(uint64_t k0, uint64_t r0, uint64_t k1, uint64_t r1) { return k0 < k1 || (k0 == k1 && r0 < r1); }

// A node record: [0,D) available, [D,2D) total, [2D] taint, [2D+1] label, [2D+2] rank << 32 | flags, padded to whole
// 32-byte lines
LT_HD constexpr int record_words(int D) { return (2 * D + 3 + 3) / 4 * 4; }

// Position p of the cycle's initial order, as the key kernel and the stable radix sort left it (sorted_key, sorted_node),
// and its node's record of RS = record_words(D) words (yk_lt_init_kernel, one position per thread; the node tables are
// column-major with leading dimension ldn)
LT_HD void init_node(int D, int p, const int64_t* __restrict__ total, const int64_t* __restrict__ avail, size_t ldn,
                     const uint64_t* __restrict__ taint, const uint64_t* __restrict__ label, const uint32_t* __restrict__ flags,
                     const uint32_t* __restrict__ rank, const uint64_t* __restrict__ sorted_key,
                     const uint32_t* __restrict__ sorted_node, int64_t* __restrict__ rec, int RS, Ent* __restrict__ ord) {
    const uint32_t n = sorted_node[p];
    int64_t* r = rec + (size_t)n * RS;
    for (int k = 0; k < D; ++k) { r[k] = avail[(size_t)k * ldn + n]; r[D + k] = total[(size_t)k * ldn + n]; }
    r[2 * D] = (int64_t)taint[n];
    r[2 * D + 1] = (int64_t)label[n];
    r[2 * D + 2] = (int64_t)(((uint64_t)rank[n] << 32) | (uint64_t)flags[n]);
    Ent e;
    e.key = sorted_key[p];
    e.rn = ((uint64_t)rank[n] << 32) | (uint64_t)n;
    ord[p] = e;
}

struct Args {
    uint32_t policy;
    double w[8];
    int64_t* rec; int RS;                  // node records (record_words / init_node)
    Ent* ord[2]; int* cur;                 // the node order, ping-pong; *cur = which buffer is current
    int nlive;
    const int64_t* a_req; size_t lda;      // ask table (column-major, as in yk_kernels.cuh)
    const uint64_t* a_tol; const uint64_t* a_need; const uint64_t* a_deny; const uint32_t* a_node;
    const uint32_t* asks; const uint32_t* meta; const uint32_t* shp; const uint32_t* sig; int B;
    uint32_t* res;                         // [B] node index or NONE
    int* hdr;                              // [H_WORDS]
    int64_t* ub;                           // [8] per-dimension upper bound of what any node can still hold (exact after a full scan)
    int insensitive;                       // 1: a failed ask does not end the batch (placement-insensitive order)
    long long* prof;                       // optional [16]: SM clocks per phase, accumulated by thread 0 (nullptr: off)
};
enum { PF_STAGE = 0, PF_SCAN, PF_WINDOW, PF_BOUND, PF_LATTICE, PF_SORT, PF_LINKS, PF_CHAIN, PF_APPLY, PF_PATCH, PF_FULLSCAN, PF_N };

// can a node in this state (available, total) take `req` once more (same fold as yk_gather_kernel: unusable -> nothing
// fits; request <= min(max(0,total), max(0,available)) on every dimension)
template <int D>
LT_HD bool fits(bool usable, const int64_t* avail, const int64_t* total, const int64_t* req) {
    if (!usable) return false;
    for (int k = 0; k < D; ++k) {
        const int64_t r = req[k];
        const int64_t t = total[k] < 0 ? 0 : total[k];
        int64_t a = avail[k];
        if (a < 0) a = 0;
        if (r > t || r > a) return false;
    }
    return true;
}

// float64 score -> sort key of a node state; one copy of the divide sequences for the whole kernel
template <int D>
LT_NI uint64_t key_of(uint32_t policy, const double* w, const int64_t* total, const int64_t* avail) {
    return yk_key_bits(yk_node_score(D, policy, w, total, avail, 1));
}

// would c * r overflow int64 (r >= 0, c >= 0)?  (a 64-bit divide costs a hundred instructions: the product's high word is free)
LT_HD bool mul_overflows(int64_t r, int64_t c) {
#if defined(__CUDA_ARCH__)
    return __umul64hi((unsigned long long)r, (unsigned long long)c) != 0ull || (long long)((unsigned long long)r * (unsigned long long)c) < 0;
#else
    return c != 0 && r > INT64_MAX / c;
#endif
}

LT_HD bool accepts(uint64_t taint, uint64_t label, uint32_t node, uint64_t tol, uint64_t need, uint64_t deny, uint32_t want) {
    if ((taint & ~tol) | (~label & need) | (label & deny)) return false;
    return want == NONE || want == node;
}

LT_HD int id_slot(uint32_t id) { return (int)((id * 2654435761u) >> 22); }   // 10 bits: HT slots

template <int D>
struct Shared {
    static constexpr int PMAX = D <= 4 ? 512 : 256;
    // ---- scalars (written inside LT_ONE or by the block reductions, read after LT_SYNC) ----
    int n, P, nrows, nshapes, cut, gstart_before_cut;
    int nbase, nvalid, nt, tdone, need_more, status, hit, esc_pos, cnt_elems, total_slots, pick;
    unsigned long long bound_key, bound_sec, pos_key;
    unsigned long long ubx[8];
    int sumv[NCAND];
    double tau[NCAND];
    int64_t sreq[SMAX * 8];       // request vector of each shape of the sub-run
    // ---- staged positions (column-major: consecutive threads touch consecutive banks) ----
    uint64_t okey[PMAX], orn[PMAX], taint[PMAX], label[PMAX];
    int64_t avail[D * PMAX], total[D * PMAX];   // [k][p]
    uint8_t usable[PMAX];
    uint8_t depth[PMAX * SMAX];   // box of the node: states c with c_s <= depth[s]
    alignas(4) uint16_t cnt[PMAX * SMAX];   // allocations of each shape the chain gave to the position
    uint32_t off[PMAX + 1];       // first slot of the node's box
    uint32_t tb[PMAX + 1];        // touched positions before p
    // ---- lattice elements: key, sec = NodeID rank << 32 | allocations in the state << 22 | slot ----
    unsigned long long e_key[LCAP], e_sec[LCAP];
    uint16_t slot_p[LCAP];        // slot -> position
    uint16_t idx_of[LCAP];        // slot -> sorted element (NO_CHILD: not below the bound)
    uint16_t child[LCAP * SMAX];  // (element, shape) -> element of the node's next state
    alignas(8) uint32_t ROOM[SMAX * FW];   // per shape: the element's node can take one more of it
    alignas(8) uint32_t BASE[FW];          // elements that are a node's initial state
    alignas(16) uint32_t F[SIGCAP * FW];   // ACCEPT rows; before the links phase and after the chain: scratch
    uint32_t scan[LCAP];
    uint64_t r_tol[SIGCAP], r_need[SIGCAP], r_deny[SIGCAP];
    uint32_t r_want[SIGCAP];
    uint8_t k_row[KCAP], k_meta[KCAP], k_ls[KCAP];
    uint32_t k_shp[KCAP], k_sig[KCAP];
    int32_t sel[KCAP];            // element taken by the ask, -1 none
    int shp_tab[HT], sig_tab[HT];
    // scratch inside F: [0, LCAP) words tmp; then the touched nodes sorted by their new (key, rn); then the same unsorted
    LT_HD uint32_t* tmp() { return F; }
    LT_HD unsigned long long* t_key() { return reinterpret_cast<unsigned long long*>(F + LCAP); }
    LT_HD unsigned long long* t_rn() { return reinterpret_cast<unsigned long long*>(F + LCAP) + PMAX; }
    LT_HD const unsigned long long* t_key() const { return reinterpret_cast<const unsigned long long*>(F + LCAP); }
    LT_HD const unsigned long long* t_rn() const { return reinterpret_cast<const unsigned long long*>(F + LCAP) + PMAX; }
    LT_HD unsigned long long* u_key() { return reinterpret_cast<unsigned long long*>(F + LCAP) + 2 * PMAX; }
    LT_HD unsigned long long* u_rn() { return reinterpret_cast<unsigned long long*>(F + LCAP) + 3 * PMAX; }
    // sort destination (before the links phase): all of F as LCAP (key, sec) pairs
    LT_HD unsigned long long* d_key() { return reinterpret_cast<unsigned long long*>(F); }
    LT_HD unsigned long long* d_sec() { return reinterpret_cast<unsigned long long*>(F) + LCAP; }
};
static_assert(SIGCAP * FW >= LCAP + 8 * 512, "scratch after the chain must fit the ACCEPT rows");
static_assert(SIGCAP * FW * 4 >= LCAP * 16, "the sort destination must fit the ACCEPT rows");
static_assert(512 * SMAX <= 2 * LCAP, "corner keys use the element arrays as scratch");

// ---- block-wide helpers (each is a sequence of LT_FOR regions: runs unchanged as plain loops on the host) -------
// exclusive prefix sum of x[0..n) (n <= 2 * THREADS) in place, total in *tot (valid on thread 0 / the host); tmp: 40 words
LT_NI void block_scan(uint32_t* x, uint32_t* tmp, int n, int* tot) {
#if LT_DEV
    const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
    const int i0 = 2 * tid, i1 = 2 * tid + 1;
    const uint32_t va = i0 < n ? x[i0] : 0u, vb = i1 < n ? x[i1] : 0u;
    uint32_t incl = va + vb;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= o) incl += u; }
    if (lane == 31) tmp[wp] = incl;
    __syncthreads();
    if (wp == 0) {
        uint32_t wv = lane < THREADS / 32 ? tmp[lane] : 0u, wi = wv;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, wi, o); if (lane >= o) wi += u; }
        tmp[lane] = wi - wv;
        if (lane == 31) tmp[32] = wi;
    }
    __syncthreads();
    const uint32_t base = tmp[wp] + incl - (va + vb);
    if (i0 < n) x[i0] = base;
    if (i1 < n) x[i1] = base + va;
    if (tid == 0) *tot = (int)tmp[32];
    __syncthreads();
#else
    uint32_t run = 0;
    for (int i = 0; i < n; ++i) { const uint32_t v = x[i]; x[i] = run; run += v; }
    *tot = (int)run;
    (void)tmp;
#endif
}
static_assert(2 * THREADS >= KCAP && 2 * THREADS >= 512, "block_scan covers two items per thread");

// ascending bitonic sort of (key, sec) pairs, n a power of two
LT_NI void block_sort(unsigned long long* key, unsigned long long* sec, int n) {
    for (int k = 2; k <= n; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            LT_FOR(x, n >> 1) {
                const int i = ((x / j) * 2 * j) + (x % j);   // lower index of the pair
                const int l = i + j;
                const bool up = (i & k) == 0;
                const unsigned long long ki = key[i], kl = key[l], si = sec[i], sl = sec[l];
                const bool gt = ki > kl || (ki == kl && si > sl);
                if (gt == up) { key[i] = kl; key[l] = ki; sec[i] = sl; sec[l] = si; }
            }
            LT_SYNC();
        }
}

// ascending sort of n <= THREADS (key, sec) pairs, result in key/sec; (bkey, bsec) is a second buffer of the same size.
// Device: one element per thread in registers; compare-exchange partners less than 32 apart swap through shuffles (no
// barrier), the others through the two buffers alternately (one barrier per such stage: 15 for 1024 elements instead of
// the 55 of the plain network above).  Host: the plain network.
LT_NI void block_sort_fast(unsigned long long* key, unsigned long long* sec, int n, unsigned long long* bkey, unsigned long long* bsec) {
#if LT_DEV
    int pn = 32;
    while (pn < n) pn <<= 1;
    const int i = threadIdx.x;
    const bool act = i < pn;
    unsigned long long k0 = (i < n) ? key[i] : KEY_INF, s0 = (i < n) ? sec[i] : KEY_INF;
    unsigned long long* buf_k[2] = {key, bkey};
    unsigned long long* buf_s[2] = {sec, bsec};
    int cur = 1;   // the first cross-warp stage writes into the second buffer (the input has been read into registers)
    __syncthreads();
    for (int k = 2; k <= pn; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            unsigned long long k1, s1;
            if (j < 32) {
                k1 = __shfl_xor_sync(0xFFFFFFFFu, k0, j); s1 = __shfl_xor_sync(0xFFFFFFFFu, s0, j);
            } else {
                if (act) { buf_k[cur][i] = k0; buf_s[cur][i] = s0; }
                __syncthreads();
                k1 = act ? buf_k[cur][i ^ j] : KEY_INF; s1 = act ? buf_s[cur][i ^ j] : KEY_INF;
                cur ^= 1;
            }
            const bool up = (i & k) == 0, lower = (i & j) == 0;
            const bool other_less = k1 < k0 || (k1 == k0 && s1 < s0);
            if ((lower == up) == other_less) { k0 = k1; s0 = s1; }   // keep the smaller when (lower == up), else the larger
        }
    __syncthreads();
    if (i < n) { key[i] = k0; sec[i] = s0; }
    __syncthreads();
#else
    int pn = 1;
    while (pn < n) pn <<= 1;
    for (int x = n; x < pn; ++x) { bkey[x - n] = 0; }   // (scratch unused on the host)
    // plain insertion of sentinels is not possible in place when n == capacity: sort the n entries directly
    for (int a2 = 1; a2 < n; ++a2) {
        const unsigned long long kk = key[a2], ss = sec[a2];
        int b2 = a2;
        for (; b2 > 0 && (key[b2 - 1] > kk || (key[b2 - 1] == kk && sec[b2 - 1] > ss)); --b2) { key[b2] = key[b2 - 1]; sec[b2] = sec[b2 - 1]; }
        key[b2] = kk; sec[b2] = ss;
    }
    (void)bsec;
#endif
}

// Sorted merge by counting: src[0, nb) is sorted, src[nb, n) is not (few entries).  Every entry counts the unsorted
// entries before it (a broadcast loop) and, when it is itself unsorted, binary-searches the sorted part: its final index.
LT_NI void block_merge_by_count(const unsigned long long* skey, const unsigned long long* ssec, int nb, int n,
                                unsigned long long* dkey, unsigned long long* dsec) {
    LT_FOR(i, n) {
        const unsigned long long k = skey[i], c = ssec[i];
        int before = 0;
        for (int x = nb; x < n; ++x) before += ent_less(skey[x], ssec[x], k, c) ? 1 : 0;
        int lo = i;
        if (i >= nb) {
            lo = 0;
            int hi = nb;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (ent_less(skey[mid], ssec[mid], k, c)) lo = mid + 1; else hi = mid; }
        }
        dkey[lo + before] = k; dsec[lo + before] = c;
    }
    LT_SYNC();
}

LT_FN void smin32(int* p, int v) {
#if LT_DEV
    atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
LT_FN void sinc16(uint16_t* p) {   // 16-bit counter inside a 32-bit word of shared memory
#if LT_DEV
    const size_t a = (size_t)p;
    uint32_t* w = (uint32_t*)(a & ~(size_t)3);
    atomicAdd(w, (a & 2) ? 0x10000u : 1u);
#else
    ++*p;
#endif
}

// Block-wide reductions into a shared word.  Every thread of the CTA calls them exactly once (outside LT_FOR) with the
// value it accumulated over its own loop iterations (the neutral element when it has none): one shuffle tree per warp,
// then at most one shared atomic per warp -- a 64-bit atomicMin on shared memory is a CAS loop, and a thousand threads
// on one address serialize for tens of microseconds.  On the host the loop has already accumulated everything.
LT_FN void red_min64(unsigned long long* p, unsigned long long v) {
#if LT_DEV
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long u = __shfl_xor_sync(0xFFFFFFFFu, v, o); v = u < v ? u : v; }
    if ((threadIdx.x & 31) == 0 && v != KEY_INF) atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
LT_FN void red_max64(unsigned long long* p, unsigned long long v) {
#if LT_DEV
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long u = __shfl_xor_sync(0xFFFFFFFFu, v, o); v = u > v ? u : v; }
    if ((threadIdx.x & 31) == 0 && v != 0ull) atomicMax(p, v);
#else
    if (v > *p) *p = v;
#endif
}
LT_FN void red_add32(int* p, int v) {
#if LT_DEV
    v = __reduce_add_sync(0xFFFFFFFFu, v);
    if ((threadIdx.x & 31) == 0 && v != 0) atomicAdd(p, v);
#else
    *p += v;
#endif
}
LT_FN void red_max32(int* p, int v) {
#if LT_DEV
    v = __reduce_max_sync(0xFFFFFFFFu, v);
    if ((threadIdx.x & 31) == 0) atomicMax(p, v);
#else
    if (v > *p) *p = v;
#endif
}
LT_FN void red_min32(int* p, int v) {
#if LT_DEV
    v = __reduce_min_sync(0xFFFFFFFFu, v);
    if ((threadIdx.x & 31) == 0) atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
// append: reserve one slot of a shared counter for every lane whose `take` is set; all 32 lanes of the warp call it
// together (loops that use it run over a multiple of 32 items: LT_FOR32)
LT_FN int warp_append(int* counter, bool take) {
#if LT_DEV
    const unsigned m = __ballot_sync(0xFFFFFFFFu, take);
    int base = 0;
    if (m && (threadIdx.x & 31) == 0) base = atomicAdd(counter, __popc(m));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    return base + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
#else
    if (!take) return 0;
    return (*counter)++;
#endif
}
// one bitmap word from 32 consecutive items (LT_FOR32 loops: item index = bit index); the host ORs bit by bit
LT_FN void put_bit(uint32_t* words, int item, bool bit) {
#if LT_DEV
    const unsigned m = __ballot_sync(0xFFFFFFFFu, bit);
    if ((threadIdx.x & 31) == 0) words[item >> 5] = m;
#else
    if ((item & 31) == 0) words[item >> 5] = 0u;
    if (bit) words[item >> 5] |= 1u << (item & 31);
#endif
}

template <typename T>
LT_FN T ldg(const T* p) {
#if LT_DEV
    return __ldcg(p);     // L2: the records and the order are rewritten by this kernel, L1 lines could be stale
#else
    return *p;
#endif
}

// ---- per node: the depth of its box along every shape for a key gap (tau - score, float) ----------------------
// d_s = how many allocations of shape s alone keep the (linearly estimated) score below tau, capped; then the box is
// shrunk (deepest side halved) until it has at most VCAP states.  A heuristic, in single precision: exactness never
// depends on the depths, only on the bound computed from the true keys just outside the boxes.  Returns the states.
LT_NI int box_of(float gap, const float* inv /*[S] 1/delta, 0 = the shape does not move the key */, int S, uint8_t* d /*[SMAX]*/) {
    int v = 1;
    for (int s = 0; s < S; ++s) {
        int x = 0;
        if (gap > 0.0f) {
            if (inv[s] > 0.0f) { const float q = gap * inv[s]; x = q >= (float)DCAP ? DCAP : (int)q; }
            else x = DCAP;
        }
        d[s] = (uint8_t)x;
        v *= x + 1;
        if (v > (1 << 24)) v = 1 << 24;
    }
    while (v > VCAP) {
        int m = 0;
        for (int s = 1; s < S; ++s) if (d[s] > d[m]) m = s;
        d[m] = (uint8_t)(d[m] >> 1);
        v = 1;
        for (int s = 0; s < S; ++s) { v *= d[s] + 1; if (v > (1 << 24)) v = 1 << 24; }   // (eight sides of 64 overflow an int)
    }
    return v;
}

// 1 / (estimated score increase of one allocation of `req` on the node): the weighted mean of req/total as yk_node_score
template <int D>
LT_NI float inv_delta_of(const double* w, const int64_t* total, const int64_t* req) {
    float u = 0.0f, tw = 0.0f;
    for (int k = 0; k < D; ++k) {
        if (!(w[k] > 0.0) || total[k] <= 0) continue;
        u += (float)w[k] * ((float)req[k] / (float)total[k]);
        tw += (float)w[k];
    }
    return (tw > 0.0f && u > 0.0f) ? tw / u : 0.0f;
}

// number of touched entries (sorted t_key/t_rn[0..nt)) that sort before (key, rn)
template <int D>
LT_NI int touched_before(const Shared<D>& s, int nt, uint64_t key, uint64_t rn) {
    const unsigned long long* tk = s.t_key();
    const unsigned long long* tr = s.t_rn();
    if (nt == 0 || !ent_less(tk[0], tr[0], key, rn)) return 0;
    if (ent_less(tk[nt - 1], tr[nt - 1], key, rn)) return nt;
    int lo = 1, hi = nt - 1;   // tk[0] < x, tk[nt-1] >= x
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ent_less(tk[mid], tr[mid], key, rn)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// ---- patch: src order minus the touched positions, merged with the touched nodes under their new keys -> dst ------
// touched positions: sub-run mode (esc_pos < 0): positions p < P with tb[p+1] > tb[p];
//                    single mode (esc_pos >= 0): exactly position esc_pos
template <int D>
LT_NI void patch_order(const Args& a, Shared<D>& s, const Ent* src, Ent* dst) {
    const int nt = s.nt, P = s.P, esc = s.esc_pos, nlive = a.nlive;
    const unsigned long long* tk = s.t_key();
    const unsigned long long* tr = s.t_rn();
    LT_FOR32(p, nlive) {
        const bool in = p < nlive;
        Ent e;
        e.key = in ? ldg(&src[p].key) : KEY_INF; e.rn = in ? ldg(&src[p].rn) : KEY_INF;
        const int ib = in ? touched_before(s, nt, e.key, e.rn) : nt;
        // the touched entries that fall between the old tuples of positions p-1 and p are written by position p
        int ibp;
#if LT_DEV
        ibp = __shfl_up_sync(0xFFFFFFFFu, ib, 1);
        if ((threadIdx.x & 31) == 0) ibp = (in && p > 0) ? touched_before(s, nt, ldg(&src[p - 1].key), ldg(&src[p - 1].rn)) : 0;
#else
        ibp = p > 0 ? touched_before(s, nt, src[p - 1].key, src[p - 1].rn) : 0;
#endif
        if (!in) continue;
        const bool touched = esc >= 0 ? (p == esc) : (p < P && s.tb[p + 1] != s.tb[p]);
        const int tbp = esc >= 0 ? (p > esc ? 1 : 0) : (p < P ? (int)s.tb[p] : nt);
        const int before = p - tbp;   // untouched old entries before position p
        for (int i = ibp; i < ib; ++i) { Ent te; te.key = tk[i]; te.rn = tr[i]; dst[i + before] = te; }
        if (!touched) dst[before + ib] = e;
        if (p == nlive - 1) {   // touched entries behind every old tuple
            const int all = before + (touched ? 0 : 1);
            for (int i = ib; i < nt; ++i) { Ent te; te.key = tk[i]; te.rn = tr[i]; dst[i + all] = te; }
        }
    }
    LT_SYNC();
}

// ---- chain: sequential first fit over the sorted elements --------------------------------------------------------
// asks [0, n) of the sub-run.  Sets sel[], tdone (asks decided), need_more (an ask found nothing below the bound: the
// sub-run ends before it -- before its gang when it is a gang member).
template <int D>
LT_NI void chain(Shared<D>& s) {
    const int n = s.n, nw = (s.nvalid + 31) >> 5;
#if LT_DEV
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        const bool h0 = lane < nw, h1 = lane + 32 < nw;
        uint32_t a0 = h0 ? s.BASE[lane] : 0u, a1 = h1 ? s.BASE[lane + 32] : 0u;   // AVAIL words lane, lane+32
        uint32_t g0 = 0, g1 = 0;   // snapshot at the gang start
        int gbeg = -1, done = n, more = 0;
        // two-deep software pipeline: the indices of ask i+1 and the candidate words of ask i are loaded ahead
        uint32_t m = s.k_meta[0];
        int sh = s.k_ls[0], row = s.k_row[0];
        uint32_t w0 = h0 ? (s.F[row * FW + lane] & s.ROOM[sh * FW + lane]) : 0u;
        uint32_t w1 = h1 ? (s.F[row * FW + lane + 32] & s.ROOM[sh * FW + lane + 32]) : 0u;
        uint32_t nm = n > 1 ? s.k_meta[1] : 0u;
        int nsh = n > 1 ? s.k_ls[1] : 0, nrow = n > 1 ? s.k_row[1] : 0;
        for (int i = 0; i < n; ++i) {
            // loads for the next two asks first: their latency hides behind this ask's ballot / shuffle
            const uint32_t xw0 = h0 ? (s.F[nrow * FW + lane] & s.ROOM[nsh * FW + lane]) : 0u;
            const uint32_t xw1 = h1 ? (s.F[nrow * FW + lane + 32] & s.ROOM[nsh * FW + lane + 32]) : 0u;
            const int i2 = i + 2 < n ? i + 2 : i;
            const uint32_t m2 = s.k_meta[i2];
            const int sh2 = s.k_ls[i2], row2 = s.k_row[i2];
            if (m & M_GSTART) { gbeg = i; g0 = a0; g1 = a1; }
            else if (!(m & M_GANG)) gbeg = -1;
            const uint32_t f0 = w0 & a0, f1 = w1 & a1;
            const uint32_t b0 = __ballot_sync(0xFFFFFFFFu, f0 != 0u);
            int e = -1;
            if (b0) {
                const int wl = __ffs((int)b0) - 1;
                const int bit = __shfl_sync(0xFFFFFFFFu, __ffs((int)f0) - 1, wl);
                if (lane == wl) a0 &= ~(1u << bit);
                e = wl * 32 + bit;
            } else {
                const uint32_t b1 = __ballot_sync(0xFFFFFFFFu, f1 != 0u);
                if (b1) {
                    const int wl = __ffs((int)b1) - 1;
                    const int bit = __shfl_sync(0xFFFFFFFFu, __ffs((int)f1) - 1, wl);
                    if (lane == wl) a1 &= ~(1u << bit);
                    e = (wl + 32) * 32 + bit;
                }
            }
            if (e < 0) {
                more = 1;
                if (gbeg >= 0) { done = gbeg; a0 = g0; a1 = g1; }   // the gang is decided as a whole by a later sub-run
                else done = i;
                break;
            }
            const int ch = s.child[e * SMAX + sh];   // every lane reads the same half-word: a broadcast
            if (ch != (int)NO_CHILD) {   // the node's next state becomes available
                const int wd = ch >> 5;
                if (wd == lane) a0 |= 1u << (ch & 31);
                else if (wd == lane + 32) a1 |= 1u << (ch & 31);
            }
            if (lane == 0) s.sel[i] = e;
            m = nm; sh = nsh; row = nrow; w0 = xw0; w1 = xw1;
            nm = m2; nsh = sh2; nrow = row2;
        }
        if (lane == 0) { s.tdone = done; s.need_more = more; }
    }
    LT_SYNC();
#else
    uint32_t av[FW], snap[FW];
    for (int w = 0; w < FW; ++w) av[w] = w < nw ? s.BASE[w] : 0u;
    int gbeg = -1, done = n, more = 0;
    for (int i = 0; i < n; ++i) {
        const uint32_t m = s.k_meta[i];
        if (m & M_GSTART) { gbeg = i; for (int w = 0; w < FW; ++w) snap[w] = av[w]; }
        else if (!(m & M_GANG)) gbeg = -1;
        const int sh = s.k_ls[i];
        const uint32_t* row = s.F + (int)s.k_row[i] * FW;
        const uint32_t* room = s.ROOM + sh * FW;
        int e = -1;
        for (int w = 0; w < nw; ++w) {
            const uint32_t f = row[w] & room[w] & av[w];
            if (f) { const int bit = __builtin_ctz(f); av[w] &= ~(1u << bit); e = w * 32 + bit; break; }
        }
        if (e < 0) {
            more = 1;
            if (gbeg >= 0) { done = gbeg; for (int w = 0; w < FW; ++w) av[w] = snap[w]; }
            else done = i;
            break;
        }
        const int ch = s.child[e * SMAX + sh];
        if (ch != (int)NO_CHILD) av[ch >> 5] |= 1u << (ch & 31);
        s.sel[i] = e;
    }
    s.tdone = done; s.need_more = more;
#endif
}

// gather a staged position's columns into contiguous arrays
template <int D>
LT_FN void load_pos(const Shared<D>& s, int p, int64_t* av, int64_t* to) {
    constexpr int PMAX = Shared<D>::PMAX;
    for (int k = 0; k < D; ++k) { av[k] = s.avail[k * PMAX + p]; to[k] = s.total[k * PMAX + p]; }
}

// ---- the batch --------------------------------------------------------------------------------------------------
template <int D>
LT_FN void lattice_batch(const Args& a, Shared<D>& s) {
    constexpr int PMAX = Shared<D>::PMAX;
    const int RS = a.RS, nlive = a.nlive, B = a.B;
    int buf = ldg(a.cur);
    int t = 0;                 // next undecided batch entry
    int status = ST_DONE;
    int subruns = 0, fullscans = 0, sorts = 0, quick = 0, escs = 0;
    long long elems = 0;
    int fresh = 0;             // 1: the previous sub-run decided nothing for entry t: decide it by a full scan
    int dead = 0;              // entry t-1 was a certain NOFIT and nothing was committed since: the same signature -> NOFIT too
    uint32_t dead_sig = 0;
    int Pwant = PMAX / 2;      // positions to scan: follows what the windows actually use
    LT_ONE s.status = ST_DONE;
    LT_FOR(i, HT) { s.shp_tab[i] = 0x7FFFFFFF; s.sig_tab[i] = 0x7FFFFFFF; }
    LT_SYNC();
#if LT_DEV
    long long prof_t = clock64();
#endif

    while (t < B && status == ST_DONE) {
        // ================= stage the asks of the sub-run =================
        const int navail = B - t < KCAP ? B - t : KCAP;
        LT_ONE { s.cut = navail; s.gstart_before_cut = 0; s.nshapes = 0; }
        LT_FOR32(i, navail) {
            const bool in = i < navail;
            const uint32_t shp = in ? ldg(&a.shp[t + i]) : 0u, sg = in ? ldg(&a.sig[t + i]) : 0u;
            if (in) { s.k_meta[i] = (uint8_t)ldg(&a.meta[t + i]); s.k_shp[i] = shp; s.k_sig[i] = sg; s.sel[i] = -1; }
            // the first entry with an id leads it: lowest index per table slot (one atomic per distinct id and warp)
#if LT_DEV
            const unsigned act = __ballot_sync(0xFFFFFFFFu, in);
            if (in) {
                const unsigned ms = __match_any_sync(act, shp), mg = __match_any_sync(act, sg);
                if ((threadIdx.x & 31) == __ffs((int)ms) - 1) atomicMin(&s.shp_tab[id_slot(shp)], i);
                if ((threadIdx.x & 31) == __ffs((int)mg) - 1) atomicMin(&s.sig_tab[id_slot(sg)], i);
            }
#else
            if (in) { smin32(&s.shp_tab[id_slot(shp)], i); smin32(&s.sig_tab[id_slot(sg)], i); }
#endif
        }
        LT_SYNC();
        // leaders (an entry whose id differs from its slot's leader leads itself: never a wrong merge, at worst a
        // duplicate shape / row); local shape numbers and rows in order of first appearance: one scan, two counters
        LT_FOR(i, navail) {
            const int ls = s.shp_tab[id_slot(s.k_shp[i])], lg = s.sig_tab[id_slot(s.k_sig[i])];
            const bool lead_s = ls == i || s.k_shp[ls] != s.k_shp[i], lead_g = lg == i || s.k_sig[lg] != s.k_sig[i];
            s.scan[i] = (lead_s ? 1u : 0u) | (lead_g ? 0x10000u : 0u);
        }
        LT_SYNC();
        { int tot; block_scan(s.scan, s.tmp(), navail, &tot); (void)tot; }
        LT_FOR(i, navail) {
            const int ls = s.shp_tab[id_slot(s.k_shp[i])], lg = s.sig_tab[id_slot(s.k_sig[i])];
            const bool lead_s = ls == i || s.k_shp[ls] != s.k_shp[i], lead_g = lg == i || s.k_sig[lg] != s.k_sig[i];
            if (lead_s) {
                const int loc = (int)(s.scan[i] & 0xFFFFu);
                if (loc >= SMAX) smin32(&s.cut, i);
                else {
                    s.k_ls[i] = (uint8_t)loc;
                    const uint32_t ask = ldg(&a.asks[t + i]);
                    for (int k = 0; k < D; ++k) s.sreq[loc * 8 + k] = ldg(&a.a_req[(size_t)k * a.lda + ask]);
                }
            }
            if (lead_g) {
                const int row = (int)(s.scan[i] >> 16);
                if (row >= SIGCAP) smin32(&s.cut, i);
                else {
                    s.k_row[i] = (uint8_t)row;
                    const uint32_t ask = ldg(&a.asks[t + i]);
                    s.r_tol[row] = ldg(&a.a_tol[ask]); s.r_need[row] = ldg(&a.a_need[ask]); s.r_deny[row] = ldg(&a.a_deny[ask]);
                    s.r_want[row] = ldg(&a.a_node[ask]);
                }
            }
        }
        LT_SYNC();
        int n = s.cut;   // everything before the first entry that would need a 9th shape / 129th row
        int my_shapes = 0, my_rows = 0;
        LT_FOR(i, navail) {
            const int ls = s.shp_tab[id_slot(s.k_shp[i])], lg = s.sig_tab[id_slot(s.k_sig[i])];
            if (i < n) {
                if (ls != i && s.k_shp[ls] == s.k_shp[i]) s.k_ls[i] = s.k_ls[ls];
                if (lg != i && s.k_sig[lg] == s.k_sig[i]) s.k_row[i] = s.k_row[lg];
                my_shapes = (int)s.k_ls[i] + 1 > my_shapes ? (int)s.k_ls[i] + 1 : my_shapes;
                my_rows = (int)s.k_row[i] + 1 > my_rows ? (int)s.k_row[i] + 1 : my_rows;
            }
        }
        red_max32(&s.nshapes, my_shapes);
        LT_ONE s.nrows = 0;
        LT_SYNC();
        red_max32(&s.nrows, my_rows);
        LT_FOR(i, navail) { s.shp_tab[id_slot(s.k_shp[i])] = 0x7FFFFFFF; s.sig_tab[id_slot(s.k_sig[i])] = 0x7FFFFFFF; }   // clean for the next sub-run
        // never cut inside a gang
        const uint32_t mnext = n < navail ? (uint32_t)s.k_meta[n] : (t + n < B ? ldg(&a.meta[t + n]) : 0u);
        if (n > 0 && (mnext & M_GANG) && !(mnext & M_GSTART)) {
            int my_g = 0;
            LT_FOR(i, n) if (s.k_meta[i] & M_GSTART) my_g = i > my_g ? i : my_g;
            red_max32(&s.gstart_before_cut, my_g);
            LT_SYNC();
            n = s.gstart_before_cut;   // 0: the gang does not fit a sub-run
        }
        if (n == 0) { status = ST_HANDOFF; break; }
        LT_ONE s.n = n;
        LT_SYNC();
        const int nrows = s.nrows, S = s.nshapes;
        const bool gang0 = (s.k_meta[0] & M_GANG) != 0;
        const int64_t* req0 = s.sreq;   // entry 0 is the first appearance of its shape: local number 0

        // ================= hopeless request: some dimension exceeds what any node has left =================
        bool hopeless = false;
        for (int k = 0; k < D; ++k) if (req0[k] > ldg(&a.ub[k])) hopeless = true;
        if (dead && s.k_sig[0] == dead_sig && !gang0) hopeless = true;   // same signature as the NOFIT just decided, same state
        if (hopeless) {
            // the first entry (its whole gang when it is a gang member) is a certain NOFIT
            int g1 = 1;
            if (gang0) while (g1 < n && (s.k_meta[g1] & M_GANG) && !(s.k_meta[g1] & M_GSTART)) ++g1;
            const uint32_t sg0 = s.k_sig[0];
            LT_FOR(i, g1) a.res[t + i] = NONE;
            LT_SYNC();
            ++quick;
            t += g1;
            dead = gang0 ? 0 : 1; dead_sig = sg0;
            if (!a.insensitive) status = ST_STOPPED;
            continue;
        }

        LT_PROF(PF_STAGE);
        if (!fresh) {
            // ================= scan: stage the first P positions =================
            const int P = nlive < Pwant ? nlive : Pwant;
            const Ent* cur = a.ord[buf];
            LT_ONE {
                s.P = P; s.nt = 0; s.esc_pos = -1; s.bound_sec = KEY_INF;
                // every element at or after the first unscanned position is unknown
                s.pos_key = P < nlive ? ldg(&cur[P].key) : KEY_INF;
                s.bound_key = s.pos_key;
                for (int c = 0; c < NCAND; ++c) s.sumv[c] = 0;
            }
            LT_FOR(p, P) {
                s.okey[p] = ldg(&cur[p].key); s.orn[p] = ldg(&cur[p].rn);
                for (int x = 0; x < SMAX; x += 2) *reinterpret_cast<uint32_t*>(&s.cnt[p * SMAX + x]) = 0u;
            }
            LT_SYNC();
            {   // the records: consecutive threads read consecutive words of one record (a few coalesced requests per
                // record instead of one request per word)
                constexpr int RW = record_words(D);   // = a.RS
                LT_FOR(x, P * RW) {
                    const int p = x / RW, w = x % RW;
                    if (w > 2 * D + 2) continue;
                    const int64_t v = ldg(&a.rec[(size_t)(uint32_t)s.orn[p] * RW + w]);
                    if (w < D) s.avail[w * PMAX + p] = v;
                    else if (w < 2 * D) s.total[(w - D) * PMAX + p] = v;
                    else if (w == 2 * D) s.taint[p] = (uint64_t)v;
                    else if (w == 2 * D + 1) s.label[p] = (uint64_t)v;
                    else { const uint32_t fl = (uint32_t)(uint64_t)v; s.usable[p] = ((fl & 1u) && !(fl & 2u)) ? 1 : 0; }
                }
                LT_SYNC();
            }
            LT_PROF(PF_SCAN);
            // ================= window: key threshold and the boxes =================
            // candidates: the keys at positions P, P/2, P/4 ...; the largest whose boxes hold at most LCAP states wins
            LT_ONE {
                for (int c = 0; c < NCAND; ++c) {
                    const int m = P >> c;
                    s.tau[c] = m >= P ? (P < nlive ? yk_key_to_score(s.pos_key) : 1e300) : yk_key_to_score(s.okey[m > 0 ? m : 0]);
                }
            }
            LT_SYNC();
            {
                int my_v[NCAND];
                for (int c = 0; c < NCAND; ++c) my_v[c] = 0;
                LT_FOR(p, P) {
                    float inv[SMAX];
                    int64_t av[D], to[D];
                    load_pos<D>(s, p, av, to);
                    for (int x = 0; x < S; ++x) inv[x] = inv_delta_of<D>(a.w, to, s.sreq + x * 8);
                    const double sc = yk_key_to_score(s.okey[p]);
                    for (int c = 0; c < NCAND; ++c) {
                        // an upper bound of the node's box (the product of the sides, capped at VCAP): never below what
                        // box_of gives, so the candidate that is picked fits
                        const double g = s.tau[c] - sc;
                        int v = 1;
                        if (s.usable[p] && g > 0.0) {
                            const float gf = g > 1e30 ? 1e30f : (float)g;
                            for (int x = 0; x < S && v < VCAP; ++x) {
                                const float q = inv[x] > 0.0f ? gf * inv[x] : (float)DCAP;
                                v *= (q >= (float)DCAP ? DCAP : (int)q) + 1;
                            }
                            if (v > VCAP) v = VCAP;
                        }
                        my_v[c] += v;
                    }
                }
                for (int c = 0; c < NCAND; ++c) red_add32(&s.sumv[c], my_v[c]);
                LT_SYNC();
            }
            LT_ONE {
                int pick = NCAND - 1;
                for (int c = NCAND - 1; c >= 0; --c) if (s.sumv[c] <= LCAP) pick = c;
                s.pick = pick;
            }
            LT_SYNC();
            const double tau = s.tau[s.pick];
            // the next sub-run scans what this window used: twice as far when the widest candidate won, half when a
            // quarter would have done
            Pwant = s.pick == 0 ? (2 * P < PMAX ? 2 * P : PMAX) : (s.pick >= 3 ? (P / 2 > 64 ? P / 2 : 64) : P);
            LT_FOR(p, P) {
                float inv[SMAX];
                uint8_t d[SMAX];
                int64_t av[D], to[D];
                load_pos<D>(s, p, av, to);
                for (int x = 0; x < S; ++x) { inv[x] = inv_delta_of<D>(a.w, to, s.sreq + x * 8); d[x] = 0; }
                const double g = tau - yk_key_to_score(s.okey[p]);
                const int v = s.usable[p] ? box_of(g > 1e30 ? 1e30f : (float)g, inv, S, d) : 1;
                for (int x = 0; x < SMAX; ++x) s.depth[p * SMAX + x] = x < S && s.usable[p] ? d[x] : 0;
                s.scan[p] = (uint32_t)v;
            }
            LT_SYNC();
            { int tot; block_scan(s.scan, s.tmp(), P, &tot); LT_ONE s.total_slots = tot; LT_SYNC(); }
            int total_slots = s.total_slots;
            if (total_slots > LCAP) {   // cannot happen with the smallest candidate unless VCAP * P/2^(NCAND-1) + P > LCAP
                LT_FOR(p, P) { for (int x = 0; x < SMAX; ++x) s.depth[p * SMAX + x] = 0; s.scan[p] = (uint32_t)p; }
                LT_SYNC();
                total_slots = P;
            }
            LT_FOR(p, P) {
                s.off[p] = s.scan[p];
                int v = 1;
                for (int x = 0; x < S; ++x) v *= s.depth[p * SMAX + x] + 1;
                for (int x = 0; x < v; ++x) s.slot_p[s.scan[p] + x] = (uint16_t)p;
            }
            LT_ONE s.off[P] = (uint32_t)total_slots;
            LT_SYNC();
            LT_PROF(PF_WINDOW);
            // ================= bound: the smallest key just outside any box =================
            // element order = (key, NodeID rank, allocations in the state); sec packs rank << 32 | allocations << 22 | slot
            unsigned long long my_bound = KEY_INF;
            LT_FOR(x, P * S) {
                const int p = x / S, sh = x % S;
                const int j = s.depth[p * SMAX + sh] + 1;
                int64_t av[D], to[D];
                load_pos<D>(s, p, av, to);
                bool ok = s.usable[p] != 0;
                for (int k = 0; k < D && ok; ++k) {
                    const int64_t r = s.sreq[sh * 8 + k];
                    if (r > 0 && mul_overflows(r, j)) ok = false;
                    av[k] -= (int64_t)(j - 1) * r;   // the state before the j-th allocation
                }
                uint64_t tk = KEY_INF;
                if (ok && fits<D>(true, av, to, s.sreq + sh * 8)) {
                    for (int k = 0; k < D; ++k) av[k] -= s.sreq[sh * 8 + k];
                    tk = key_of<D>(a.policy, a.w, to, av);
                    my_bound = tk < my_bound ? tk : my_bound;
                }
                if (x < LCAP) s.e_key[x] = tk; else s.e_sec[x - LCAP] = tk;   // scratch until the elements are written (P * S <= 2 LCAP)
            }
            red_min64(&s.bound_key, my_bound);
            LT_SYNC();
            {
                const uint64_t bk0 = s.bound_key;
                unsigned long long my_sec = KEY_INF;
                LT_FOR(x, P * S) if ((x < LCAP ? s.e_key[x] : s.e_sec[x - LCAP]) == bk0 && bk0 != KEY_INF) {
                    const int p = x / S, sh = x % S;
                    const unsigned long long v = ((s.orn[p] >> 32) << 32) | ((unsigned long long)(s.depth[p * SMAX + sh] + 1) << 22);
                    my_sec = v < my_sec ? v : my_sec;
                }
                LT_ONE if (P < nlive && s.pos_key == bk0) { const unsigned long long v = (ldg(&cur[P].rn) >> 32) << 32; my_sec = v < my_sec ? v : my_sec; }
                red_min64(&s.bound_sec, my_sec);
                LT_SYNC();
            }
            const uint64_t bk = s.bound_key, bs = s.bound_sec;
            LT_PROF(PF_BOUND);
            // ================= lattice: the states of every box =================
            // bases (state 0) keep their position order; the other states are appended and merged in afterwards
            LT_FOR(p, P) {
                const uint64_t sec = ((s.orn[p] >> 32) << 32) | (unsigned long long)s.off[p];
                s.scan[p] = (s.usable[p] && ent_less(s.okey[p], sec, bk, bs)) ? 1u : 0u;
            }
            LT_SYNC();
            { int nb; block_scan(s.scan, s.tmp(), P, &nb); LT_ONE { s.nbase = nb; s.cnt_elems = nb; } LT_SYNC(); }
            const int nbase = s.nbase;
            LT_FOR(p, P) {
                const uint64_t sec = ((s.orn[p] >> 32) << 32) | (unsigned long long)s.off[p];
                if (s.usable[p] && ent_less(s.okey[p], sec, bk, bs)) { const int x = (int)s.scan[p]; s.e_key[x] = s.okey[p]; s.e_sec[x] = sec; }
            }
            LT_SYNC();
            LT_FOR32(x, total_slots) {
                bool take = false;
                uint64_t key = 0, sec = 0;
                if (x < total_slots && x != (int)s.off[s.slot_p[x]]) {   // (the base of a box was written above)
                    const int p = s.slot_p[x];
                    int loc = x - (int)s.off[p];
                    int64_t av[D], to[D];
                    load_pos<D>(s, p, av, to);
                    int csum = 0;
                    bool ok = true;
                    // the state is reachable iff its allocations fit one after the other (any order: the tests are monotone)
                    for (int sh = 0; sh < S; ++sh) {
                        const int dim = s.depth[p * SMAX + sh] + 1;
                        const int c = loc % dim;
                        loc /= dim;
                        csum += c;
                        for (int k = 0; k < D && ok; ++k) {
                            const int64_t r = s.sreq[sh * 8 + k];
                            if (c > 0 && r > 0) {
                                if (mul_overflows(r, c) || r > (to[k] < 0 ? 0 : to[k])) { ok = false; break; }
                                av[k] -= (int64_t)c * r;
                                if (av[k] < 0) { ok = false; break; }
                            }
                        }
                    }
                    if (ok) {
                        key = key_of<D>(a.policy, a.w, to, av);
                        sec = ((s.orn[p] >> 32) << 32) | ((unsigned long long)csum << 22) | (unsigned long long)x;
                        take = ent_less(key, sec, bk, bs);
                    }
                }
                const int y = warp_append(&s.cnt_elems, take);
                if (take) { s.e_key[y] = key; s.e_sec[y] = sec; }
            }
            LT_SYNC();
            const int nvalid = s.cnt_elems;
            LT_PROF(PF_LATTICE);
            if (nvalid > nbase) {   // deeper states interleave with the bases (which are in order already)
                if (nvalid <= THREADS) {
                    block_sort_fast(s.e_key, s.e_sec, nvalid, s.d_key(), s.d_sec());
                } else if (nvalid - nbase <= ECNT) {
                    block_merge_by_count(s.e_key, s.e_sec, nbase, nvalid, s.d_key(), s.d_sec());
                    LT_FOR(x, nvalid) { s.e_key[x] = s.d_key()[x]; s.e_sec[x] = s.d_sec()[x]; }
                    LT_SYNC();
                } else {
                    int pn = 1;
                    while (pn < nvalid) pn <<= 1;
                    LT_FOR(x, pn - nvalid) { s.e_key[nvalid + x] = KEY_INF; s.e_sec[nvalid + x] = KEY_INF; }
                    LT_SYNC();
                    block_sort(s.e_key, s.e_sec, pn);
                }
                ++sorts;
            }
            LT_ONE s.nvalid = nvalid;
            elems += nvalid;
            LT_PROF(PF_SORT);
            // ================= links: slot -> element, then per element its ROOM / BASE / ACCEPT bits and children =================
            LT_FOR(x, total_slots) s.idx_of[x] = NO_CHILD;
            LT_SYNC();
            LT_FOR(e, nvalid) s.idx_of[(int)(s.e_sec[e] & 0x3FFFFFu)] = (uint16_t)e;
            LT_SYNC();
            LT_FOR32(e, (nvalid + 63) & ~63) {   // whole 64-bit words of every bitmap get written
                const bool in = e < nvalid;
                const int slot = in ? (int)(s.e_sec[e] & 0x3FFFFFu) : 0;
                const int p = in ? (int)s.slot_p[slot] : 0;
                int loc = slot - (int)s.off[p];
                put_bit(s.BASE, e, in && loc == 0);
                int64_t av[D], to[D];
                load_pos<D>(s, p, av, to);
                unsigned long long cvec = 0;   // the state, one byte per shape
                for (int q = 0; q < S; ++q) {
                    const int dim = s.depth[p * SMAX + q] + 1;
                    const int c = loc % dim;
                    loc /= dim;
                    cvec |= (unsigned long long)c << (8 * q);
                    for (int k = 0; k < D; ++k) av[k] -= (int64_t)c * s.sreq[q * 8 + k];
                }
                int stride = 1;
                for (int sh = 0; sh < S; ++sh) {
                    const bool room = in && fits<D>(true, av, to, s.sreq + sh * 8);
                    put_bit(s.ROOM + sh * FW, e, room);
                    const int c = (int)((cvec >> (8 * sh)) & 0xFFu), dep = s.depth[p * SMAX + sh];
#if !LT_DEV && defined(YK_LT_DEBUG)
                    if (in && room && c < dep && slot + stride >= (int)s.off[s.P]) { fprintf(stderr, "DBG e=%d slot=%d stride=%d p=%d loc0=%d S=%d sh=%d c=%d dep=%d off=%u off1=%u total=%u nvalid=%d depths=%d,%d,%d,%d cvec=%llx\n", e, slot, stride, p, slot-(int)s.off[p], S, sh, c, dep, s.off[p], s.off[p+1], s.off[s.P], nvalid, s.depth[p*SMAX],s.depth[p*SMAX+1],s.depth[p*SMAX+2],s.depth[p*SMAX+3], cvec); abort(); }
#endif
                    if (in) s.child[e * SMAX + sh] = (room && c < dep) ? s.idx_of[slot + stride] : NO_CHILD;
                    stride *= dep + 1;
                }
                const uint64_t tnt = s.taint[p], lbl = s.label[p];
                const uint32_t node = (uint32_t)s.orn[p];
                for (int r = 0; r < nrows; ++r)
                    put_bit(s.F + r * FW, e, in && accepts(tnt, lbl, node, s.r_tol[r], s.r_need[r], s.r_deny[r], s.r_want[r]));
            }
            LT_SYNC();
            LT_PROF(PF_LINKS);
            // ================= chain =================
            chain<D>(s);
            ++subruns;
            const int tdone = s.tdone;
            LT_PROF(PF_CHAIN);
            if (tdone == 0) {   // nothing decided: the first entry needs the full scan
                fresh = 1;
                continue;
            }
            // ================= apply =================
            LT_FOR(i, tdone) {
                const int e = s.sel[i];
                const int p = s.slot_p[(int)(s.e_sec[e] & 0x3FFFFFu)];
                a.res[t + i] = (uint32_t)s.orn[p];
                sinc16(&s.cnt[p * SMAX + s.k_ls[i]]);
            }
            LT_SYNC();
            LT_FOR(p, P) {
                uint32_t any = 0;
                for (int x = 0; x < S; ++x) any |= s.cnt[p * SMAX + x];
                s.scan[p] = any ? 1u : 0u;
            }
            LT_SYNC();
            { int nt; block_scan(s.scan, s.tmp(), P, &nt); LT_ONE s.nt = nt; LT_SYNC(); }
            const int nt = s.nt;
            {
                unsigned long long* uk = s.u_key();
                unsigned long long* ur = s.u_rn();
                LT_FOR(p, P) {
                    s.tb[p] = s.scan[p];
                    uint32_t any = 0;
                    for (int x = 0; x < S; ++x) any |= s.cnt[p * SMAX + x];
                    if (any) {
                        int64_t na[D], to[D];
                        load_pos<D>(s, p, na, to);
                        int64_t* r = a.rec + (size_t)(uint32_t)s.orn[p] * RS;
                        for (int k = 0; k < D; ++k) {
                            int64_t v = na[k];
                            for (int x = 0; x < S; ++x) v -= (int64_t)s.cnt[p * SMAX + x] * s.sreq[x * 8 + k];
                            na[k] = v; r[k] = v;
                        }
                        const uint64_t nk = key_of<D>(a.policy, a.w, to, na);
                        if (nk == YK_KEY_NAN) s.status = ST_NAN;
                        const int x = (int)s.scan[p];
                        uk[x] = nk; ur[x] = s.orn[p];
                    }
                }
                LT_ONE { s.tb[P] = (uint32_t)nt; }
                LT_SYNC();
                if (s.status == ST_NAN) { status = ST_NAN; break; }
                LT_FOR(x, nt) { s.t_key()[x] = uk[x]; s.t_rn()[x] = ur[x]; }
                LT_SYNC();
                block_sort_fast(s.t_key(), s.t_rn(), nt, uk, ur);   // touched nodes by their new keys
            }
            LT_PROF(PF_APPLY);
            patch_order<D>(a, s, a.ord[buf], a.ord[buf ^ 1]);
            LT_PROF(PF_PATCH);
            buf ^= 1;
            t += tdone;
            dead = 0;
            continue;
        }

        // ================= full scan: exact first fit of entry t over the whole order =================
        fresh = 0;
        ++fullscans;
        {
            const Ent* cur = a.ord[buf];
            const uint64_t tol = s.r_tol[0], need = s.r_need[0], deny = s.r_deny[0];
            const uint32_t want = s.r_want[0];
            LT_ONE { s.hit = nlive; for (int k = 0; k < D; ++k) s.ubx[k] = 0; }
            LT_SYNC();
            for (int base = 0; base < nlive && s.hit == nlive; base += THREADS * 4) {
                const int lim = nlive - base < THREADS * 4 ? nlive - base : THREADS * 4;
                unsigned long long my_ub[D];
                for (int k = 0; k < D; ++k) my_ub[k] = 0;
                int my_hit = nlive;
                LT_FOR(x, lim) {
                    const int p = base + x;
                    const uint64_t rn = ldg(&cur[p].rn);
                    const uint32_t node = (uint32_t)rn;
                    const int64_t* r = a.rec + (size_t)node * RS;
                    int64_t av[D], to[D];
                    for (int k = 0; k < D; ++k) { av[k] = ldg(&r[k]); to[k] = ldg(&r[D + k]); }
                    const uint32_t fl = (uint32_t)(uint64_t)ldg(&r[2 * D + 2]);
                    const bool usable = (fl & 1u) && !(fl & 2u);
                    if (usable)
                        for (int k = 0; k < D; ++k) {
                            const int64_t aa = av[k] < 0 ? 0 : av[k], tt = to[k] < 0 ? 0 : to[k];
                            const unsigned long long cc = (unsigned long long)(aa < tt ? aa : tt);
                            my_ub[k] = cc > my_ub[k] ? cc : my_ub[k];
                        }
                    if (fits<D>(usable, av, to, req0) &&
                        accepts((uint64_t)ldg(&r[2 * D]), (uint64_t)ldg(&r[2 * D + 1]), node, tol, need, deny, want))
                        my_hit = p < my_hit ? p : my_hit;
                }
                for (int k = 0; k < D; ++k) red_max64(&s.ubx[k], my_ub[k]);
                red_min32(&s.hit, my_hit);
                LT_SYNC();
            }
            const int hit = s.hit;
            if (hit == nlive) {   // certain NOFIT (of the whole gang when the entry leads one); every node was seen: the
                int g1 = 1;       // capacity bound is exact now
                if (gang0) while (g1 < n && (s.k_meta[g1] & M_GANG) && !(s.k_meta[g1] & M_GSTART)) ++g1;
                const uint32_t sg0 = s.k_sig[0];
                LT_FOR(i, g1) a.res[t + i] = NONE;
                LT_ONE { for (int k = 0; k < D; ++k) a.ub[k] = (int64_t)s.ubx[k]; }
                LT_SYNC();
                t += g1;
                dead = gang0 ? 0 : 1; dead_sig = sg0;
                if (!a.insensitive) status = ST_STOPPED;
                LT_PROF(PF_FULLSCAN);
                continue;
            }
            // a gang whose first member fits somewhere but that could not be placed from the front of the order: the
            // host path decides it (it can roll a partly placed gang back)
            if (gang0) { status = ST_HANDOFF; break; }
            // commit the ask to the node at position `hit`
            ++escs;
            LT_ONE {
                const uint64_t rn = ldg(&cur[hit].rn);
                const uint32_t node = (uint32_t)rn;
                int64_t* r = a.rec + (size_t)node * RS;
                int64_t na[D], to[D];
                for (int k = 0; k < D; ++k) { na[k] = ldg(&r[k]) - req0[k]; to[k] = ldg(&r[D + k]); r[k] = na[k]; }
                const uint64_t nk = key_of<D>(a.policy, a.w, to, na);
                if (nk == YK_KEY_NAN) s.status = ST_NAN;
                s.t_key()[0] = nk; s.t_rn()[0] = rn;
                s.nt = 1; s.esc_pos = hit; s.P = 0;
                a.res[t] = node;
            }
            LT_SYNC();
            if (s.status == ST_NAN) { status = ST_NAN; break; }
            patch_order<D>(a, s, a.ord[buf], a.ord[buf ^ 1]);
            buf ^= 1;
            t += 1;
            dead = 0;
            LT_PROF(PF_FULLSCAN);
        }
    }
    LT_ONE {
        *a.cur = buf;
        a.hdr[H_CONSUMED] = t;
        a.hdr[H_STATUS] = status;
        a.hdr[H_SUBRUNS] += subruns; a.hdr[H_FULLSCANS] += fullscans; a.hdr[H_SORTS] += sorts;
        a.hdr[H_ELEMS] += (int)(elems > 0x7FFFFFFF ? 0x7FFFFFFF : elems); a.hdr[H_QUICK] += quick; a.hdr[H_ESC] += escs;
    }
    LT_SYNC();
}

}  // namespace yklt
