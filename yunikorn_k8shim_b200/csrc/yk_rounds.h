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
// Spent nodes leave the order: a node that is unusable, or whose capacity on some dimension is below the stretch's smallest
// request there, can take no ask of the stretch.  Left in place, a full node at the front would make every round a single
// step.  They are parked unsorted and merged back under their final keys when the stretch ends.
//
// A guard ends the stretch when rounds stay short (fewer than `guard` asks per pass on average after the first 16 passes):
// what has been decided stands, and the rest of the cycle goes to the host commit.
#pragma once
#include <stdint.h>
#include "yk_lattice.h"

namespace ykrd {

using yklt::Ent;
using yklt::KEY_INF;
using yklt::NONE;
using yklt::THREADS;
typedef unsigned long long u64;

constexpr int WCAP = THREADS;           // candidates per round: one per thread
constexpr int SIDE = 2 * WCAP;          // re-keyed entries kept sorted in shared memory before they go back into the order
constexpr int GUARD_PASSES = 16;        // passes before the guard looks at the asks per pass
// the guard's asks per pass: a pass costs 24-40 us at 2 000-10 000 nodes (H100, DESIGN.md §6.3), the host path 0.2-0.3 us
// per ask, so a stretch that averages fewer asks per pass costs several times what the host path would
constexpr int GUARD = 32;

// hdr[] words: asks decided, yklt::ST_*, passes, single steps, nodes that left the order
enum { R_CONSUMED = 0, R_STATUS = 1, R_PASSES = 2, R_SINGLES = 3, R_SPENT = 4, R_WORDS = 5 };

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
    uint32_t* res;                         // [B] node index or NONE
    int* hdr;                              // [R_WORDS]
    int window;                            // candidates per round, 1..WCAP
    int guard;                             // asks per pass below which the stretch ends (0: never)
    long long* prof;                       // optional [RP_N]: SM clocks per phase, accumulated by thread 0 (nullptr: off)
};
enum { RP_EDGES = 0, RP_CAND, RP_SCAN, RP_APPLY, RP_SORT, RP_MERGE, RP_SINGLE, RP_N };   // stretch set-up + restore, then per round

struct Shared {
    int m, n_new, n_sp, hit, nan, keep;
    int64_t minreq[8];
    u64 ck[WCAP], cr[WCAP];                // candidate j: the new entry of S[j] after ask i+j (KEY_INF: S[j] rejects it)
    u64 ek[WCAP], er[WCAP];                // S[j] itself: the first W entries of order + side list
    uint8_t fs[WCAP];                      // ... 1 when it comes from the side list
    u64 pk[WCAP], pr[WCAP];                // exclusive prefix minimum of (ck, cr); sort scratch afterwards
    u64 tk[WCAP], tr[WCAP];                // the taken nodes' new entries that stay in the order, then sorted
    u64 wk[32], wr[32];                    // per-warp partials of the prefix minimum
    uint32_t scan[WCAP];
    uint32_t tmp[40];
    u64 lk[2][SIDE], lr[2][SIDE];          // the side list, ping-pong
};
static_assert(THREADS <= 1024 && WCAP <= THREADS, "one candidate per thread, at most 32 warps");

LT_FN bool ent_lt(u64 k0, u64 r0, u64 k1, u64 r1) { return yklt::ent_less(k0, r0, k1, r1); }

// exclusive prefix minimum of the pairs (k, r)[0, n), n <= THREADS, into (pk, pr); (KEY_INF, KEY_INF) is neutral
LT_NI void block_prefmin(Shared& s, int n) {
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
    if (i < n) { s.pk[i] = fa; s.pr[i] = fb; }
    __syncthreads();
#else
    u64 ma = KEY_INF, mb = KEY_INF;
    for (int i = 0; i < n; ++i) {
        s.pk[i] = ma; s.pr[i] = mb;
        if (ent_lt(s.ck[i], s.cr[i], ma, mb)) { ma = s.ck[i]; mb = s.cr[i]; }
    }
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

// can node n (record r) take ask `ask`?  The lattice kernel's test: usable, masks, node name, capacity on every dimension
template <int D>
LT_FN bool accepts_ask(const Args& a, const int64_t* r, uint32_t n, uint32_t ask, int64_t* req) {
    for (int k = 0; k < D; ++k) req[k] = a.a_req[(size_t)k * a.lda + ask];
    const uint32_t fl = (uint32_t)(uint64_t)r[2 * D + 2];
    return yklt::fits<D>((fl & 1u) && !(fl & 2u), r, r + D, req) &&
           yklt::accepts((uint64_t)r[2 * D], (uint64_t)r[2 * D + 1], n, a.a_tol[ask], a.a_need[ask], a.a_deny[ask], a.a_node[ask]);
}

// the side list goes back into the order: ord[buf][hd, hd + n) merged with it into ord[buf ^ 1][0, n + nl)
LT_FN void flush_side(const Args& a, Shared& s, int& buf, int& hd, int& n, int& nl, int lb) {
    if (nl == 0) return;
    merge_into(a.ord[buf] + hd, n, 0, 0, s.lk[lb], s.lr[lb], nl, a.ord[buf ^ 1]);
    buf ^= 1; hd = 0; n += nl; nl = 0;
}

// ---- the stretch -------------------------------------------------------------------------------------------------
template <int D>
LT_FN void rounds_stretch(const Args& a, Shared& s) {
    const int RS = a.RS, nlive = a.nlive, B = a.B;
    int buf = *a.cur;
    int t = 0, status = yklt::ST_DONE, passes = 0, singles = 0;
#if LT_DEV
    long long prof_t = clock64();
#endif

    // ---- the smallest request of the stretch per dimension (requests of an ask that reaches a commit are >= 0) ----
    LT_ONE { for (int k = 0; k < 8; ++k) s.minreq[k] = INT64_MAX; s.n_sp = 0; s.keep = 0; s.nan = 0; }
    LT_SYNC();
    for (int k = 0; k < D; ++k) {
        u64 my = KEY_INF;
        LT_FOR(i, B) { const int64_t v = a.a_req[(size_t)k * a.lda + a.asks[i]]; const u64 c = v < 0 ? 0ull : (u64)v; my = c < my ? c : my; }
        yklt::red_min64(reinterpret_cast<u64*>(&s.minreq[k]), my);
    }
    LT_SYNC();

    // ---- spent nodes leave the order (stable for the rest) ----
    int n_act = 0;
    for (int base = 0; base < nlive; base += THREADS) {
        const int lim = nlive - base < THREADS ? nlive - base : THREADS;
        LT_FOR32(x, lim) {
            const bool in = x < lim;
            const Ent e = in ? a.ord[buf][base + x] : Ent{0, 0};
            const bool sp = in && spent_of<D>(a.rec + (size_t)(uint32_t)e.rn * RS, s.minreq);
            if (in) s.scan[x] = sp ? 0u : 1u;
            const int y = yklt::warp_append(&s.n_sp, sp);
            if (sp) a.spent[y] = e;
        }
        LT_SYNC();
        { int tot; yklt::block_scan(s.scan, s.tmp, lim, &tot); LT_ONE s.keep = tot; LT_SYNC(); }
        LT_FOR(x, lim) {
            const Ent e = a.ord[buf][base + x];
            const bool keep = (x + 1 < lim ? s.scan[x + 1] : (uint32_t)s.keep) != s.scan[x];
            if (keep) a.ord[buf ^ 1][n_act + (int)s.scan[x]] = e;
        }
        n_act += s.keep;
        LT_SYNC();
    }
    buf ^= 1;
    // The order is ord[buf][hd, hd + n_act) merged with the side list (s.lk / s.lr[lb], nl entries, sorted): a round takes
    // a prefix of both, its new entries join the side list, and only a full side list is merged back into the order --
    // the order itself is never rewritten for one round, only its head moves.
    int hd = 0, nl = 0, lb = 0;
    LT_PROF(RP_EDGES);

    while (t < B) {
        const int left = B - t;
        int W = a.window < left ? a.window : left;
        W = W < n_act + nl ? W : n_act + nl;
        const int wm = W < n_act ? W : n_act, wl = W < nl ? W : nl;
        LT_ONE { s.m = W; s.n_new = 0; s.keep = 0; }
        {   // ---- S[0, W): the first W entries of order + side list ----
            const Ent* A = a.ord[buf] + hd;
            const u64* lk = s.lk[lb];
            const u64* lr = s.lr[lb];
            LT_FOR(x, wm) { const Ent e = A[x]; s.pk[x] = e.key; s.pr[x] = e.rn; }
            LT_SYNC();
            LT_FOR(x, wm) {
                const int r = x + new_before(lk, lr, nl, s.pk[x], s.pr[x]);
                if (r < W) { s.ek[r] = s.pk[x]; s.er[r] = s.pr[x]; s.fs[r] = 0; }
            }
            LT_FOR(y, wl) {
                const int r = y + new_before(s.pk, s.pr, wm, lk[y], lr[y]);
                if (r < W) { s.ek[r] = lk[y]; s.er[r] = lr[y]; s.fs[r] = 1; }
            }
            LT_SYNC();
        }
        // ---- candidates: S[j] for ask t+j ----
        LT_FOR(j, W) {
            const uint32_t n = (uint32_t)s.er[j];
            const int64_t* r = a.rec + (size_t)n * RS;
            int64_t req[D], na[D];
            const bool ok = accepts_ask<D>(a, r, n, a.asks[t + j], req);
            u64 key = KEY_INF;
            if (ok) {
                for (int k = 0; k < D; ++k) na[k] = r[k] - req[k];
                key = yklt::key_of<D>(a.policy, a.w, r + D, na);
            }
            s.ck[j] = key; s.cr[j] = ok ? s.er[j] : KEY_INF;
        }
        LT_SYNC();
        LT_PROF(RP_CAND);
        block_prefmin(s, W);
        {   // m: the first candidate that rejects its ask or does not sort before the new entries ahead of it
            int my = W;
            LT_FOR(j, W) if (s.cr[j] == KEY_INF || !ent_lt(s.ek[j], s.cr[j], s.pk[j], s.pr[j])) my = j < my ? j : my;
            yklt::red_min32(&s.m, my);
            LT_SYNC();
        }
        const int m = s.m;
        LT_PROF(RP_SCAN);
        ++passes;
        bool moved = false;   // the order was rewritten into the other buffer
        if (m > 0) {
            int my_nan = 0, my_side = 0;
            LT_FOR(j, m) { if (s.ck[j] == KEY_INF) my_nan = 1; my_side += s.fs[j]; }
            yklt::red_max32(&s.nan, my_nan);
            yklt::red_add32(&s.keep, my_side);
            LT_SYNC();
            if (s.nan) { status = yklt::ST_NAN; break; }
            const int ml = s.keep, mm = m - ml;   // taken from the side list / from the order
            // ---- apply; the new entries stay in the order or leave it ----
            LT_FOR32(j, m) {
                bool stay = false;
                Ent ne{0, 0};
                if (j < m) {
                    const uint32_t n = (uint32_t)s.cr[j];
                    int64_t* r = a.rec + (size_t)n * RS;
                    const uint32_t ask = a.asks[t + j];
                    for (int k = 0; k < D; ++k) r[k] -= a.a_req[(size_t)k * a.lda + ask];
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
            yklt::block_sort_fast(s.tk, s.tr, nt, s.pk, s.pr);
            LT_PROF(RP_SORT);
            hd += mm; n_act -= mm;
            const u64* ok_ = s.lk[lb] + ml;
            const u64* or_ = s.lr[lb] + ml;
            const int no = nl - ml;   // what is left of the side list
            if (no + nt <= SIDE) {   // the new entries join the side list
                u64* dk = s.lk[lb ^ 1];
                u64* dr = s.lr[lb ^ 1];
                LT_FOR(y, no) { const int p = y + new_before(s.tk, s.tr, nt, ok_[y], or_[y]); dk[p] = ok_[y]; dr[p] = or_[y]; }
                LT_FOR(i, nt) { const int p = i + new_before(ok_, or_, no, s.tk[i], s.tr[i]); dk[p] = s.tk[i]; dr[p] = s.tr[i]; }
                LT_SYNC();
                lb ^= 1; nl = no + nt;
            } else {   // the side list is full: it goes back into the order, the new entries start the next one
                merge_into(a.ord[buf] + hd, n_act, 0, 0, ok_, or_, no, a.ord[buf ^ 1]);
                buf ^= 1; hd = 0; n_act += no;
                LT_FOR(i, nt) { s.lk[lb][i] = s.tk[i]; s.lr[lb][i] = s.tr[i]; }
                LT_SYNC();
                nl = nt;
            }
            LT_PROF(RP_MERGE);
            t += m;
        } else {
            // ---- one exact step: the first position of the whole order that accepts ask t ----
            ++singles;
            flush_side(a, s, buf, hd, n_act, nl, lb);
            LT_ONE s.hit = n_act;
            LT_SYNC();
            Ent* src = a.ord[buf] + hd;
            const uint32_t ask = a.asks[t];
            int hit = n_act;
            for (int base = 0; base < n_act && hit == n_act; base += THREADS) {
                const int lim = n_act - base < THREADS ? n_act - base : THREADS;
                int my = n_act;
                LT_FOR(x, lim) {
                    const uint32_t n = (uint32_t)src[base + x].rn;
                    int64_t req[D];
                    if (accepts_ask<D>(a, a.rec + (size_t)n * RS, n, ask, req)) my = base + x < my ? base + x : my;
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
                    int64_t na[D];
                    for (int k = 0; k < D; ++k) na[k] = r[k] - a.a_req[(size_t)k * a.lda + ask];
                    Ent ne; ne.key = yklt::key_of<D>(a.policy, a.w, r + D, na); ne.rn = e.rn;
                    if (ne.key == KEY_INF) s.nan = 1;
                    else {
                        for (int k = 0; k < D; ++k) r[k] = na[k];
                        a.res[t] = n;
                        if (spent_of<D>(r, s.minreq)) { a.spent[s.n_sp++] = ne; s.n_new = 0; }
                        else { s.tk[0] = ne.key; s.tr[0] = ne.rn; s.n_new = 1; }
                    }
                }
                LT_SYNC();
                if (s.nan) { status = yklt::ST_NAN; break; }
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
        if (a.guard > 0 && passes >= GUARD_PASSES && t < B && (long long)t < (long long)a.guard * passes) {
            status = yklt::ST_HANDOFF;
            break;
        }
    }

    // ---- the side list and the spent nodes return, the latter under their final keys, a sorted chunk at a time ----
    flush_side(a, s, buf, hd, n_act, nl, lb);
    const int n_sp = s.n_sp;
    for (int base = 0; base < n_sp; base += WCAP) {
        const int nt = n_sp - base < WCAP ? n_sp - base : WCAP;
        LT_FOR(x, nt) { const Ent e = a.spent[base + x]; s.tk[x] = e.key; s.tr[x] = e.rn; }
        LT_SYNC();
        yklt::block_sort_fast(s.tk, s.tr, nt, s.pk, s.pr);
        merge_into(a.ord[buf] + hd, n_act, 0, 0, s.tk, s.tr, nt, a.ord[buf ^ 1]);
        hd = 0;
        n_act += nt;
        buf ^= 1;
    }
    LT_PROF(RP_EDGES);
    LT_ONE {
        *a.cur = buf;
        a.hdr[R_CONSUMED] = t;
        a.hdr[R_STATUS] = status;
        a.hdr[R_PASSES] = passes;
        a.hdr[R_SINGLES] = singles;
        a.hdr[R_SPENT] = n_sp;
    }
    LT_SYNC();
}

}  // namespace ykrd
