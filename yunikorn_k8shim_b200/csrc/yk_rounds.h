// yk_rounds.h -- the device-resident ordered commit for MASK-FREE stretches ("round commit"), single source like
// yk_lattice.h: nvcc builds it into yk_rounds_kernel (one persistent CTA, yk_rounds.cuh), g++ into plain loops for the CPU
// test suite (tests/host/device_shim.cpp).
//
// What it replaces: the same one-allocation-per-pass loop as yk_lattice.h under the `fair` node sort, for a stretch of
// consecutive asks in a placement-insensitive order that carry no masks (no required / forbidden labels, no node name, every
// taint tolerated): only capacity can make a node reject such an ask.
//
// Why a round is parallel.  Let S be the node order, ascending by (key, NodeID rank).  Suppose asks i, i+1, ... take the
// front nodes S[0], S[1], ... in turn.  Then ask i+j takes S[j] exactly when
//   (a) S[j] accepts ask i+j, and
//   (b) S[j] sorts before the smallest of the new (key, rank) entries that S[0..j-1] got from their allocations:
// every node ahead of S[j] has been taken, every untaken node behind it sorts after it, and (b) says every re-keyed node
// sorts after it too.  No assumption on the scores is needed.  A round evaluates W candidates at once (the acceptance test
// and the new key of S[j] for ask i+j), takes an exclusive prefix minimum of the new entries, and decides the asks before
// the first candidate that fails (a) or (b) -- m of them.  m = 0 means the front node rejects ask i: that ask is decided
// by one exact step, the first accepting position of the whole order (or NOFIT in place).  The m taken nodes are applied,
// their new entries sorted and kept in a side list in shared memory; the order is the untaken rest merged with that list,
// and only a full side list is merged back into the order -- one rewrite of the order per several rounds, not per round.
//
// Sub-rounds.  A staged window leaves the order: it is kept sorted in shared memory, and every entry it holds sorts before
// the first entry that was not staged (the fence) -- the window is an exact prefix of the order.  After a round, the
// untaken rest of the window merged with the new entries that sort before the fence is again an exact prefix (everything
// else sorts after the fence), so the next round runs on it without reading the order or the side list; new entries at or
// after the fence join the side list.  Only a window shorter than REFILL is topped up from the order and the side list.
//
// Spent nodes leave the order: a node that is unusable, or whose capacity on some dimension is below the stretch's smallest
// request there, can take no ask of the stretch.  Left in place, a full node at the front would make every round a single
// step.  They are parked unsorted and merged back under their final keys when the stretch ends.
//
// A guard ends the stretch when rounds stay short (fewer than `guard` asks per pass on average after the first 16 passes):
// what has been decided stands, and the rest of the cycle goes to the host commit.
#pragma once
#include <assert.h>
#include <stdint.h>
#include "yk_lattice.h"
#include "yk_spec.h"
#if !LT_DEV
#include <vector>
#endif

namespace ykrd {

using yklt::Ent;
using yklt::KEY_INF;
using yklt::NONE;
using yklt::THREADS;
typedef unsigned long long u64;

constexpr int WCAP = THREADS;           // candidates per round: one per thread
constexpr int SIDE = 2 * WCAP;          // re-keyed entries kept sorted in shared memory before they go back into the order
// a window shorter than this is topped up before the next round (DESIGN.md §6.3: on config 2, rounds decide ~240 asks, and
// a window that has run down to REFILL entries caps the next round below that)
constexpr int REFILL = WCAP / 2;
constexpr int GUARD_PASSES = 16;        // passes before the guard looks at the asks per pass
// the guard's asks per pass: a pass costs 24-40 us at 2 000-10 000 nodes (H100, DESIGN.md §6.3), the host path 0.2-0.3 us
// per ask, so a stretch that averages fewer asks per pass costs several times what the host path would
constexpr int GUARD = 32;
constexpr int PUBLISH_PASSES = 8;       // passes per publication of the decided count (Args::prog), a power of two

// hdr[] words: asks decided, yklt::ST_* or ST_ABORTED, passes, single steps, nodes that left the order
enum { R_CONSUMED = 0, R_STATUS = 1, R_PASSES = 2, R_SINGLES = 3, R_SPENT = 4, R_WORDS = 5 };
// a speculative launch (Args::go) that did not run, or stopped because the host set Args::abort: the host reads nothing
// it wrote
constexpr int ST_ABORTED = 4;

struct Args {
    uint32_t policy;
    double w[8];
    int64_t* rec; int RS;                  // node records (yk_lattice.h Args::rec)
    Ent* ord[2]; int* cur;                 // the node order, ping-pong; *cur = which buffer is current
    int nlive;
    Ent* spent;                            // [nlive] scratch: the entries of the nodes that left the order
    const int64_t* a_req; size_t lda;      // ask table (column-major)
    const uint64_t* a_tol; const uint64_t* a_need; const uint64_t* a_deny; const uint32_t* a_node;
    const uint32_t* asks; int B;           // the stretch
    int64_t* sreq;                         // [B][D] scratch: the stretch's requests in stretch order, written at its start
                                           // (host: one is allocated when it is null)
    uint32_t* res;                         // [B] node index or NONE
    int* hdr;                              // [R_WORDS]
    volatile int* prog;                    // device: asks decided so far, published every PUBLISH_PASSES passes for the host,
                                           // which settles them while the stretch goes on (nullptr: off); never read here
    int window;                            // candidates per round, 1..WCAP
    int guard;                             // asks per pass below which the stretch ends (0: never)
    long long* prof;                       // optional [RP_N]: SM clocks per phase, accumulated by thread 0 (nullptr: off)
    // a speculative launch (yk_spec.h), started before the host knows the stretch: go[ykspec::W_STATUS] is the screen's
    // status and go[ykspec::W_COUNT] replaces B; the kernel returns at once unless the status is ykspec::GO and the node
    // order's NaN flag (*nan) is clear.  abort: a host word in mapped memory, read with each publication; once set, the
    // stretch ends with ST_ABORTED.  All three nullptr for a launch of a known stretch.
    const uint32_t* go; const int* nan; const volatile int* abort;
};
// stretch set-up + restore, then per round; RP_FRESH counts the window's fresh stagings (not clocks)
enum { RP_EDGES = 0, RP_CAND, RP_SCAN, RP_APPLY, RP_SORT, RP_MERGE, RP_SINGLE, RP_FRESH, RP_N };

struct Shared {
    int m, n_new, n_sp, hit, nan, keep, stop, B;   // B: the stretch's length (Args::B, or the speculative launch's count)
    int ls;                                // the side list's entries this pass staged: its first live entry until the pass ends
    int status, singles, passes;           // for the header (kept in registers for the exits, they spill)
    long long prof_t;
    int64_t minreq[8];
    u64 fk, fr;                            // the fence: the first entry of order + side list behind the window (KEY_INF: none)
    u64 ck[WCAP], cr[WCAP];                // candidate j: the new entry of S[j] after ask i+j (KEY_INF: S[j] rejects it)
    // ping-pong: (vk, vr)[vb] is the window, S[j] = (vk, vr)[vb][j], an exact prefix of the order; the other pair is the
    // pass's scratch (staging, +1 for the fence; the exclusive prefix minimum of (ck, cr); the sort) and then the next window.
    // (One pair less keeps the block under 132 KB, which leaves the L1 room for the window's node records.)
    u64 vk[2][WCAP + 1], vr[2][WCAP + 1];
    u64 tk[WCAP], tr[WCAP];                // the taken nodes' new entries that stay in the order, then sorted
    u64 wk[32], wr[32];                    // per-warp partials of the prefix minimum
    uint32_t tmp[40];
    u64 lk[2][SIDE], lr[2][SIDE];          // the side list, ping-pong
};
static_assert(THREADS <= 1024 && WCAP <= THREADS, "one candidate per thread, at most 32 warps");

LT_FN bool ent_lt(u64 k0, u64 r0, u64 k1, u64 r1) { return yklt::ent_less(k0, r0, k1, r1); }

// exclusive prefix minimum of the pairs (ck, cr)[0, n), n <= THREADS, into (pk, pr); (KEY_INF, KEY_INF) is neutral
LT_FN void block_prefmin(Shared& s, int n, u64* pk, u64* pr) {
#if LT_DEV
    const int i = threadIdx.x, lane = i & 31, wp = i >> 5;
    u64 a = i < n ? s.ck[i] : KEY_INF, b = i < n ? s.cr[i] : KEY_INF;
    for (int o = 1; o < 32; o <<= 1) {
        const u64 ua = __shfl_up_sync(0xFFFFFFFFu, a, o), ub = __shfl_up_sync(0xFFFFFFFFu, b, o);
        if (lane >= o && ent_lt(ua, ub, a, b)) { a = ua; b = ub; }
    }
    if (lane == 31) { s.wk[wp] = a; s.wr[wp] = b; }
    __syncthreads();
    if (wp == 0) {   // exclusive minimum over the warps before
        u64 x = lane < THREADS / 32 ? s.wk[lane] : KEY_INF, y = lane < THREADS / 32 ? s.wr[lane] : KEY_INF;
        for (int o = 1; o < 32; o <<= 1) {
            const u64 ux = __shfl_up_sync(0xFFFFFFFFu, x, o), uy = __shfl_up_sync(0xFFFFFFFFu, y, o);
            if (lane >= o && ent_lt(ux, uy, x, y)) { x = ux; y = uy; }
        }
        u64 ex = __shfl_up_sync(0xFFFFFFFFu, x, 1), ey = __shfl_up_sync(0xFFFFFFFFu, y, 1);
        if (lane == 0) { ex = KEY_INF; ey = KEY_INF; }
        s.wk[lane] = ex; s.wr[lane] = ey;
    }
    __syncthreads();
    u64 ea = __shfl_up_sync(0xFFFFFFFFu, a, 1), eb = __shfl_up_sync(0xFFFFFFFFu, b, 1);
    if (lane == 0) { ea = KEY_INF; eb = KEY_INF; }
    u64 fa = s.wk[wp], fb = s.wr[wp];
    if (ent_lt(ea, eb, fa, fb)) { fa = ea; fb = eb; }
    if (i < n) { pk[i] = fa; pr[i] = fb; }
    __syncthreads();
#else
    u64 ma = KEY_INF, mb = KEY_INF;
    for (int i = 0; i < n; ++i) {
        pk[i] = ma; pr[i] = mb;
        if (ent_lt(s.ck[i], s.cr[i], ma, mb)) { ma = s.ck[i]; mb = s.cr[i]; }
    }
#endif
}

// ascending sort of the round's n <= THREADS new entries (key, sec), result in key/sec; (bkey, bsec) a second buffer.
// Device, over the next power of two pn >= n only (a round of config 2 keeps ~320 new entries: 16 of the 32 warps sort,
// the others only meet the barriers): each warp sorts its 32 entries in registers (a shuffle network, no barrier), then
// runs of w merge pairwise into runs of 2w through shared memory, one barrier per level -- an entry's place in the merged
// run is its index in its own run plus the entries of the other run before it (a binary search; ties, which only the
// padding has, go to the first run).  Host: the same function as the lattice kernel's.
LT_FN void sort_new(u64* key, u64* sec, int n, u64* bkey, u64* bsec) {
#if LT_DEV
    int pn = 32;
    while (pn < n) pn <<= 1;
    const int i = threadIdx.x;
    const bool act = i < pn;   // whole warps
    u64 k0 = i < n ? key[i] : KEY_INF, s0 = i < n ? sec[i] : KEY_INF;
    if (act)
        for (int k = 2; k <= 32; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) {
                const u64 k1 = __shfl_xor_sync(0xFFFFFFFFu, k0, j), s1 = __shfl_xor_sync(0xFFFFFFFFu, s0, j);
                const bool up = (i & k & 31) == 0, lower = (i & j) == 0;   // (every warp's run ascends)
                const bool other_less = k1 < k0 || (k1 == k0 && s1 < s0);
                if ((lower == up) == other_less) { k0 = k1; s0 = s1; }   // keep the smaller when (lower == up), else the larger
            }
    u64 *sk = key, *ss = sec, *dk = bkey, *ds = bsec;
    if (act) { sk[i] = k0; ss[i] = s0; }   // (each thread reads and writes only its own index until the barrier)
    __syncthreads();
    for (int w = 32; w < pn; w <<= 1) {
        if (act) {
            const int base = i & ~(2 * w - 1);
            const bool second = (i & w) != 0;
            const u64* ok = sk + (second ? base : base + w);   // the other run
            const u64* os = ss + (second ? base : base + w);
            int lo = 0, hi = w;   // entries of the other run before this one (the first run wins ties)
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                const bool before = second ? !ent_lt(k0, s0, ok[mid], os[mid]) : ent_lt(ok[mid], os[mid], k0, s0);
                if (before) lo = mid + 1; else hi = mid;
            }
            const int p = base + (i & (w - 1)) + lo;
            dk[p] = k0; ds[p] = s0;
        }
        u64* t = sk; sk = dk; dk = t;
        t = ss; ss = ds; ds = t;
        __syncthreads();
        if (act) { k0 = sk[i]; s0 = ss[i]; }   // (dk was last read before that barrier)
    }
    if (sk != key && i < n) { key[i] = k0; sec[i] = s0; }
    __syncthreads();
#else
    yklt::block_sort_fast(key, sec, n, bkey, bsec);
#endif
}

// number of entries of the sorted (tk, tr)[0, nt) before (key, rn)
LT_FN int new_before(const u64* tk, const u64* tr, int nt, u64 key, u64 rn) {
    if (nt == 0 || !ent_lt(tk[0], tr[0], key, rn)) return 0;
    if (ent_lt(tk[nt - 1], tr[nt - 1], key, rn)) return nt;
    int lo = 1, hi = nt - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ent_lt(tk[mid], tr[mid], key, rn)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// dst = src[0, n) without the positions [lo, hi), merged with the sorted (tk, tr)[0, nt).  Every kept position writes
// itself and the new entries that fall between it and the kept position before it; the last one also those behind it.
// Device: a warp's 32 consecutive positions are sorted, so lanes 0 and 31 bound the new entries the warp can see and the
// other lanes search only between them; the count before the previous position comes from the lane next door (the
// binary searches over shared memory are what a merge of 10 000 positions costs).
LT_NI void merge_into(const Ent* src, int n, int lo, int hi, const u64* tk, const u64* tr, int nt, Ent* dst) {
    const int gone = hi - lo, kept = n - gone;
    const int last = hi == n ? lo - 1 : n - 1;
    if (kept == 0) {
        LT_FOR(i, nt) { Ent e; e.key = tk[i]; e.rn = tr[i]; dst[i] = e; }
    }
    LT_FOR32(p, n) {
        const bool in = p < n;
        Ent e;
        e.key = in ? src[p].key : KEY_INF; e.rn = in ? src[p].rn : KEY_INF;
        const int q = (p == hi && gone > 0) ? lo - 1 : p - 1;   // the kept position before p
#if LT_DEV
        const int lane = threadIdx.x & 31;
        int wlo = lane == 0 ? new_before(tk, tr, nt, e.key, e.rn) : 0;
        int whi = lane == 31 ? new_before(tk, tr, nt, e.key, e.rn) : 0;
        wlo = __shfl_sync(0xFFFFFFFFu, wlo, 0);
        whi = __shfl_sync(0xFFFFFFFFu, whi, 31);
        const int ib = wlo + new_before(tk + wlo, tr + wlo, whi - wlo, e.key, e.rn);
        int ibp = __shfl_up_sync(0xFFFFFFFFu, ib, 1);
        if (lane == 0 || q != p - 1) ibp = (in && q >= 0) ? new_before(tk, tr, nt, src[q].key, src[q].rn) : 0;
#else
        const int ib = new_before(tk, tr, nt, e.key, e.rn);
        const int ibp = q >= 0 ? new_before(tk, tr, nt, src[q].key, src[q].rn) : 0;
#endif
        if (!in || (p >= lo && p < hi)) continue;
        const int before = p >= hi ? p - gone : p;               // kept positions before p
        for (int i = ibp; i < ib; ++i) { Ent t; t.key = tk[i]; t.rn = tr[i]; dst[i + before] = t; }
        dst[before + ib] = e;
        if (p == last) for (int i = ib; i < nt; ++i) { Ent t; t.key = tk[i]; t.rn = tr[i]; dst[i + before + 1] = t; }
    }
    LT_SYNC();
}

// a node in this state can take no ask of the stretch: unusable, or below the smallest request on some dimension
template <int D>
LT_FN bool spent_of(const int64_t* r, const int64_t* minreq) {
    const uint32_t fl = (uint32_t)(uint64_t)r[2 * D + 2];
    if (!(fl & 1u) || (fl & 2u)) return true;
    for (int k = 0; k < D; ++k) {
        const int64_t t = r[D + k] < 0 ? 0 : r[D + k], a = r[k] < 0 ? 0 : r[k];
        if (minreq[k] > (t < a ? t : a)) return true;
    }
    return false;
}

// the staged request of stretch position i
template <int D>
LT_FN void req_of(const Args& a, int i, int64_t* q) {
    for (int k = 0; k < D; ++k) q[k] = a.sreq[(size_t)i * D + k];
}

// Can node n (record r) take request q of stretch position i?  The lattice kernel's test without the masks and the node
// name: a stretch routed here has no required or forbidden labels and no node name, and tolerates every live taint
// (yklt::round_eligible), so only the flags and the capacity decide.  The host checks that the masks would have agreed.
template <int D>
LT_FN bool takes(const Args& a, const int64_t* r, uint32_t n, int i, const int64_t* q) {
    const uint32_t fl = (uint32_t)(uint64_t)r[2 * D + 2];
    bool ok = (fl & 1u) && !(fl & 2u);
    for (int k = 0; k < D; ++k) {
        const int64_t t = r[D + k] < 0 ? 0 : r[D + k], v = r[k] < 0 ? 0 : r[k];
        ok = ok && q[k] <= t && q[k] <= v;
    }
#if !LT_DEV
    if (ok) {
        const uint32_t ask = a.asks[i];
        assert(yklt::accepts((uint64_t)r[2 * D], (uint64_t)r[2 * D + 1], n, a.a_tol[ask], a.a_need[ask], a.a_deny[ask], a.a_node[ask]));
    }
#endif
    (void)a; (void)n; (void)i;
    return ok;
}

// the key of node record r once it has taken request q: yk_node_score inlined on values in registers (yklt::key_of is
// a call that puts its arrays in local memory), the same double operations in the same order, so the same bits
template <int D>
LT_FN u64 key_after(const Args& a, const int64_t* r, const int64_t* q) {
    int64_t av[D], tt[D];
    for (int k = 0; k < D; ++k) { av[k] = r[k] - q[k]; tt[k] = r[D + k]; }
    return yk_key_bits(yk_node_score(D, a.policy, a.w, tt, av, 1));
}

// the window and the side list (s.lk / s.lr[lb][ls, ls + nl)) go back into the order.  The window sorts before everything
// else, so it goes in front: without a side list into the consumed positions before the head when they are enough,
// otherwise ord[buf][hd, hd + n) merged with the side list into ord[buf ^ 1][nv, nv + n + nl), behind the window.
LT_FN void restore(const Args& a, Shared& s, int& buf, int& hd, int& n, int& nl, int lb, int ls, int& nv, int vb) {
    if (nl == 0 && nv == 0) return;
    if (nl == 0 && nv <= hd) {
        Ent* dst = a.ord[buf] + hd - nv;
        LT_FOR(x, nv) { Ent e; e.key = s.vk[vb][x]; e.rn = s.vr[vb][x]; dst[x] = e; }
        LT_SYNC();
        hd -= nv; n += nv; nv = 0;
        return;
    }
    Ent* dst = a.ord[buf ^ 1];
    LT_FOR(x, nv) { Ent e; e.key = s.vk[vb][x]; e.rn = s.vr[vb][x]; dst[x] = e; }
    merge_into(a.ord[buf] + hd, n, 0, 0, s.lk[lb] + ls, s.lr[lb] + ls, nl, dst + nv);   // (ends with a barrier)
    buf ^= 1; hd = 0; n += nl + nv; nl = 0; nv = 0;
}

// Thread 0, after a barrier that follows the res writes of the asks [0, t): t for the host.  Called at the top of every
// PUBLISH_PASSES-th pass; the passes after the last one come with the header.  The system-scope fence orders every thread's
// res writes (made visible to thread 0 by the barrier) before the count, so a host that reads t with acquire semantics
// reads their results too.  The fence waits for the pass's res writes to reach host memory, ~3 us on H100 (config 2: the
// candidate phase grew by 6.5 k SM clocks per pass when every pass published), so it is paid once per 8 passes.
// A speculative launch also reads its abort word here into s.stop, which every thread reads at the end of the same pass, so
// the whole block leaves together.
LT_FN void publish(const Args& a, Shared& s, int t) {
#if LT_DEV
    if (threadIdx.x == 0) {
        if (a.prog) { __threadfence_system(); *a.prog = t; }
        if (a.abort) s.stop = *a.abort;
    }
#else
    (void)a; (void)s; (void)t;
#endif
}

// ---- the stretch -------------------------------------------------------------------------------------------------
template <int D>
LT_FN void stretch(const Args& a, Shared& s) {
    const int RS = a.RS, nlive = a.nlive;
    // (every thread reads the same words: the whole block returns, or none of it)
    if (a.go && (a.go[ykspec::W_STATUS] != ykspec::GO || *a.nan)) {
        LT_ONE { a.hdr[R_CONSUMED] = 0; a.hdr[R_STATUS] = ST_ABORTED; a.hdr[R_PASSES] = 0; a.hdr[R_SINGLES] = 0; a.hdr[R_SPENT] = 0; }
        return;
    }
    int buf = *a.cur;
    int t = 0, passes = 0;
#if LT_DEV
    long long& prof_t = s.prof_t;   // thread 0's clock; in shared memory, not in a register held through every round
    LT_ONE prof_t = clock64();
#endif

    // ---- the stretch's requests staged in stretch order, and the smallest per dimension (requests of an ask that
    // reaches a commit are >= 0) ----
    // (the stretch's length is read from s.B where it is used: held in a register through every round, it spills)
    LT_ONE { for (int k = 0; k < 8; ++k) s.minreq[k] = INT64_MAX; s.n_sp = 0; s.keep = 0; s.nan = 0; s.stop = 0; s.status = yklt::ST_DONE; s.singles = 0; s.passes = 0; s.B = a.go ? (int)a.go[ykspec::W_COUNT] : a.B; }
    LT_SYNC();
    {
        u64 my[D];
        for (int k = 0; k < D; ++k) my[k] = KEY_INF;
        LT_FOR(i, s.B) {
            const uint32_t ask = a.asks[i];
            for (int k = 0; k < D; ++k) {
                const int64_t v = a.a_req[(size_t)k * a.lda + ask];
                a.sreq[(size_t)i * D + k] = v;
                const u64 c = v < 0 ? 0ull : (u64)v;
                my[k] = c < my[k] ? c : my[k];
            }
        }
        for (int k = 0; k < D; ++k) yklt::red_min64(reinterpret_cast<u64*>(&s.minreq[k]), my[k]);
    }
    LT_SYNC();

    // ---- spent nodes leave the order (stable for the rest) ----
    uint32_t* scan = reinterpret_cast<uint32_t*>(s.ck);   // (no candidate yet)
    int n_act = 0;
    for (int base = 0; base < nlive; base += THREADS) {
        const int lim = nlive - base < THREADS ? nlive - base : THREADS;
        LT_FOR32(x, lim) {
            const bool in = x < lim;
            const Ent e = in ? a.ord[buf][base + x] : Ent{0, 0};
            const bool sp = in && spent_of<D>(a.rec + (size_t)(uint32_t)e.rn * RS, s.minreq);
            if (in) scan[x] = sp ? 0u : 1u;
            const int y = yklt::warp_append(&s.n_sp, sp);
            if (sp) a.spent[y] = e;
        }
        LT_SYNC();
        yklt::block_scan(scan, s.tmp, lim, &s.keep);   // (the total straight into shared memory: a local's address puts it in local memory)
        LT_FOR(x, lim) {
            const Ent e = a.ord[buf][base + x];
            const bool keep = (x + 1 < lim ? scan[x + 1] : (uint32_t)s.keep) != scan[x];
            if (keep) a.ord[buf ^ 1][n_act + (int)scan[x]] = e;
        }
        n_act += s.keep;
        LT_SYNC();
    }
    buf ^= 1;
    // The order is the window (s.vk / s.vr[vb], nv entries: an exact prefix, see the top of the file), then
    // ord[buf][hd, hd + n_act) merged with the side list (s.lk / s.lr[lb][0, nl), sorted; [s.ls, s.ls + nl) from a staging
    // to the end of its pass, which moves it back to the front), both at or behind the fence.  A staging moves the front of
    // those two into the window, a round takes a prefix of the window, its new entries join the window or the side list,
    // and only a full side list is merged back into the order -- the order itself is never rewritten for one round, only
    // its head moves.
    int hd = 0, nl = 0, lb = 0, nv = 0;
    bool nan_round = false;   // the stretch ended in a round's NaN check, before the window moved
    LT_PROF(RP_EDGES);

    while (t < s.B) {
        if ((passes & (PUBLISH_PASSES - 1)) == 0) publish(a, s, t);   // (the res writes so far are behind the barriers that ended their passes)
        const int left = s.B - t;
        const int cap = a.window < left ? a.window : left;   // the entries a round can use
        const int vb = passes & 1;   // the window's buffer: every pass moves the window into the other one or empties it
        // entries to stage: the window is topped up to cap (or to every live entry) when it is shorter than REFILL
        const int ns = nv < cap && nv < REFILL ? (cap < nv + n_act + nl ? cap : nv + n_act + nl) - nv : 0;
        const int W = nv + ns < cap ? nv + ns : cap;
        LT_ONE { s.m = W; s.n_new = 0; s.keep = 0; s.ls = 0; if (ns > 0) { s.fk = KEY_INF; s.fr = KEY_INF; } }
        u64* pk = s.vk[vb ^ 1];   // the pass's scratch
        u64* pr = s.vr[vb ^ 1];
        int64_t q[D];   // a candidate's request: D consecutive words of the staged requests, not a gather from the ask table
        if (ns > 0) {   // ---- a fresh staging: the first ns entries of order + side list join the window, the next is the fence ----
            const Ent* A = a.ord[buf] + hd;
            const u64* lk = s.lk[lb];
            const u64* lr = s.lr[lb];
            const int wm = ns < n_act ? ns + 1 : n_act, wl = ns < nl ? ns + 1 : nl;
            u64* vk = s.vk[vb] + nv;
            u64* vr = s.vr[vb] + nv;
            LT_FOR(x, wm) { const Ent e = A[x]; pk[x] = e.key; pr[x] = e.rn; }
            LT_SYNC();
            int mine = 0, side = 0;   // window entries from the order, from the side list
            LT_FOR(x, wm) {
                const int r = x + new_before(lk, lr, nl, pk[x], pr[x]);
                if (r < ns) { vk[r] = pk[x]; vr[r] = pr[x]; ++mine; }
                else if (r == ns) { s.fk = pk[x]; s.fr = pr[x]; }
            }
            LT_FOR(y, wl) {
                const int r = y + new_before(pk, pr, wm, lk[y], lr[y]);
                if (r < ns) { vk[r] = lk[y]; vr[r] = lr[y]; ++side; }
                else if (r == ns) { s.fk = lk[y]; s.fr = lr[y]; }
            }
            yklt::red_add32(&s.keep, mine);
            yklt::red_add32(&s.ls, side);
            LT_SYNC();
            hd += s.keep; n_act -= s.keep; nl -= s.ls; nv += ns;
#if LT_DEV
            if (a.prof && threadIdx.x == 0) a.prof[RP_FRESH] += 1;
#endif
        }
        // ---- candidates: S[j] for ask t+j ----
        LT_FOR(j, W) {
            req_of<D>(a, t + j, q);
            const u64 rn = s.vr[vb][j];
            const uint32_t n = (uint32_t)rn;
            const int64_t* r = a.rec + (size_t)n * RS;
            const bool ok = takes<D>(a, r, n, t + j, q);
            s.ck[j] = ok ? key_after<D>(a, r, q) : KEY_INF; s.cr[j] = ok ? rn : KEY_INF;
        }
        LT_SYNC();
        LT_PROF(RP_CAND);
        block_prefmin(s, W, pk, pr);
        {   // m: the first candidate that rejects its ask or does not sort before the new entries ahead of it
            int my = W;
            LT_FOR(j, W) if (s.cr[j] == KEY_INF || !ent_lt(s.vk[vb][j], s.cr[j], pk[j], pr[j])) my = j < my ? j : my;
            yklt::red_min32(&s.m, my);
            LT_SYNC();
        }
        const int m = s.m;
        LT_PROF(RP_SCAN);
        ++passes;
        LT_ONE s.passes = passes;
        bool moved = false;   // the order was rewritten into the other buffer
        if (m > 0) {
            int my_nan = 0;
            LT_FOR(j, m) if (s.ck[j] == KEY_INF) my_nan = 1;
            yklt::red_max32(&s.nan, my_nan);
            LT_SYNC();
            if (s.nan) { LT_ONE s.status = yklt::ST_NAN; nan_round = true; break; }
            // ---- apply; the new entries stay in the order or leave it ----
            LT_FOR32(j, m) {
                bool stay = false;
                Ent ne{0, 0};
                if (j < m) {
                    req_of<D>(a, t + j, q);   // (reloaded: kept in registers across the prefix minimum, it spills)
                    const uint32_t n = (uint32_t)s.cr[j];
                    int64_t* r = a.rec + (size_t)n * RS;
                    for (int k = 0; k < D; ++k) r[k] -= q[k];
                    a.res[t + j] = n;
                    ne.key = s.ck[j]; ne.rn = s.cr[j];
                    stay = !spent_of<D>(r, s.minreq);
                }
                const int y = yklt::warp_append(&s.n_new, stay);
                if (stay) { s.tk[y] = ne.key; s.tr[y] = ne.rn; }
                const int z = yklt::warp_append(&s.n_sp, j < m && !stay);
                if (j < m && !stay) a.spent[z] = ne;
            }
            LT_SYNC();
            LT_PROF(RP_APPLY);
            const int nt = s.n_new;
            sort_new(s.tk, s.tr, nt, pk, pr);
            LT_PROF(RP_SORT);
            // ---- the next window: its untaken rest merged with the new entries before the fence ----
            const int nb = new_before(s.tk, s.tr, nt, s.fk, s.fr), nr = nv - m;
            {
                const u64* rk = s.vk[vb] + m;
                const u64* rr = s.vr[vb] + m;
                u64* dk = pk;   // (the sort's scratch until the barrier that ended it)
                u64* dr = pr;
                LT_FOR(y, nr) { const int p = y + new_before(s.tk, s.tr, nb, rk[y], rr[y]); dk[p] = rk[y]; dr[p] = rr[y]; }
                LT_FOR(i, nb) { const int p = i + new_before(rk, rr, nr, s.tk[i], s.tr[i]); dk[p] = s.tk[i]; dr[p] = s.tr[i]; }
            }
            // ---- the others join the side list ----
            const u64* nk = s.tk + nb;
            const u64* nr_ = s.tr + nb;
            const int na = nt - nb;
            const u64* ok_ = s.lk[lb] + s.ls;
            const u64* or_ = s.lr[lb] + s.ls;
            if (na == 0) {   // (the side list back to the front of a buffer)
                if (s.ls > 0) {
                    LT_FOR(y, nl) { s.lk[lb ^ 1][y] = ok_[y]; s.lr[lb ^ 1][y] = or_[y]; }
                    lb ^= 1;
                }
                LT_SYNC();
            } else if (nl + na <= SIDE) {
                u64* dk = s.lk[lb ^ 1];
                u64* dr = s.lr[lb ^ 1];
                LT_FOR(y, nl) { const int p = y + new_before(nk, nr_, na, ok_[y], or_[y]); dk[p] = ok_[y]; dr[p] = or_[y]; }
                LT_FOR(i, na) { const int p = i + new_before(ok_, or_, nl, nk[i], nr_[i]); dk[p] = nk[i]; dr[p] = nr_[i]; }
                LT_SYNC();
                lb ^= 1; nl += na;
            } else {   // the side list is full: it goes back into the order, the new entries start the next one
                merge_into(a.ord[buf] + hd, n_act, 0, 0, ok_, or_, nl, a.ord[buf ^ 1]);
                buf ^= 1; hd = 0; n_act += nl;
                LT_FOR(i, na) { s.lk[lb][i] = nk[i]; s.lr[lb][i] = nr_[i]; }
                LT_SYNC();
                nl = na;
            }
            nv = nr + nb;
            LT_PROF(RP_MERGE);
            t += m;
        } else {
            // ---- one exact step: the first position of the whole order that accepts ask t ----
            LT_ONE ++s.singles;
            restore(a, s, buf, hd, n_act, nl, lb, s.ls, nv, vb);
            LT_ONE s.hit = n_act;
            LT_SYNC();
            Ent* src = a.ord[buf] + hd;
            req_of<D>(a, t, q);
            int hit = n_act;
            for (int base = 0; base < n_act && hit == n_act; base += THREADS) {
                const int lim = n_act - base < THREADS ? n_act - base : THREADS;
                int my = n_act;
                LT_FOR(x, lim) {
                    const uint32_t n = (uint32_t)src[base + x].rn;
                    if (takes<D>(a, a.rec + (size_t)n * RS, n, t, q)) my = base + x < my ? base + x : my;
                }
                yklt::red_min32(&s.hit, my);
                LT_SYNC();
                hit = s.hit;
                LT_SYNC();   // everyone has read it before the next chunk lowers it
            }
            if (hit == n_act) {   // NOFIT: the ask fails in place (placement-insensitive order)
                LT_ONE a.res[t] = NONE;
                LT_SYNC();
            } else {
                LT_ONE {
                    const Ent e = src[hit];
                    const uint32_t n = (uint32_t)e.rn;
                    int64_t* r = a.rec + (size_t)n * RS;
                    Ent ne; ne.key = key_after<D>(a, r, q); ne.rn = e.rn;
                    if (ne.key == KEY_INF) s.nan = 1;
                    else {
                        for (int k = 0; k < D; ++k) r[k] -= q[k];
                        a.res[t] = n;
                        if (spent_of<D>(r, s.minreq)) { a.spent[s.n_sp++] = ne; s.n_new = 0; }
                        else { s.tk[0] = ne.key; s.tr[0] = ne.rn; s.n_new = 1; }
                    }
                }
                LT_SYNC();
                if (s.nan) { LT_ONE s.status = yklt::ST_NAN; break; }
                const int nt = s.n_new;
                hd += 1 - nt;   // (the end of the order stays where it is)
                merge_into(src, n_act, hit, hit + 1, s.tk, s.tr, nt, a.ord[buf ^ 1] + hd);
                n_act += nt - 1;
                moved = true;
            }
            t += 1;
            LT_PROF(RP_SINGLE);
        }
        if (moved) buf ^= 1;
        // a publishing pass reads s.stop after its last barrier; thread 0 writes it next at the top of the next publishing
        // pass, behind the barriers of the passes between
        if (((passes - 1) & (PUBLISH_PASSES - 1)) == 0 && s.stop) { LT_ONE s.status = ST_ABORTED; break; }
        if (a.guard > 0 && passes >= GUARD_PASSES && t < s.B && (long long)t < (long long)a.guard * passes) {
            LT_ONE s.status = yklt::ST_HANDOFF;
            break;
        }
    }

    LT_ONE { a.hdr[R_CONSUMED] = t; a.hdr[R_PASSES] = s.passes; }

    // ---- the window, the side list and the spent nodes return, the last under their final keys, a sorted chunk at a time ----
    restore(a, s, buf, hd, n_act, nl, lb, nan_round ? s.ls : 0, nv, (s.passes & 1) ^ (nan_round ? 1 : 0));
    const int n_sp = s.n_sp;
    for (int base = 0; base < n_sp; base += WCAP) {
        const int nt = n_sp - base < WCAP ? n_sp - base : WCAP;
        LT_FOR(x, nt) { const Ent e = a.spent[base + x]; s.tk[x] = e.key; s.tr[x] = e.rn; }
        LT_SYNC();
        sort_new(s.tk, s.tr, nt, s.vk[0], s.vr[0]);   // (the window is back in the order)
        merge_into(a.ord[buf] + hd, n_act, 0, 0, s.tk, s.tr, nt, a.ord[buf ^ 1]);
        hd = 0;
        n_act += nt;
        buf ^= 1;
    }
    LT_PROF(RP_EDGES);
    LT_ONE {
        *a.cur = buf;
        a.hdr[R_STATUS] = s.status;
        a.hdr[R_SINGLES] = s.singles;
        a.hdr[R_SPENT] = n_sp;
    }
    LT_SYNC();
}

template <int D>
LT_FN void rounds_stretch(const Args& a, Shared& s) {
#if LT_DEV
    stretch<D>(a, s);
#else
    if (a.sreq) { stretch<D>(a, s); return; }
    std::vector<int64_t> own((size_t)(a.B > 0 ? a.B : 1) * D);   // a caller that brings no staging buffer
    Args b = a;
    b.sreq = own.data();
    stretch<D>(b, s);
#endif
}

}  // namespace ykrd
