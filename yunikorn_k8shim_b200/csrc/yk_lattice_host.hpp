// yk_lattice_host.hpp -- host side of the device commit (yk_lattice.h, yk_uniform.h): the per-entry meta words the kernel
// reads, the test that decides whether a cycle may use the device commit at all, and the driver around the kernels (the
// batch loop, the segment loop, a uniform run's attempts; settle and fill_batch, which the host commit uses too).  No CUDA
// in here: csrc/yk_engine.cu drives the kernels with it and tests/host/lattice_shim.cpp drives their per-item code with it.
#pragma once
#include <chrono>
#include <cstdint>
#include <unordered_map>
#include <vector>

#include "../../include/ykgpu.h"
#include "yk_commit.hpp"
#include "yk_lattice.h"
#include "yk_orderer.hpp"
#include "yk_uniform.h"

namespace yk {

// after a failure in a placement-sensitive order, probe with short batches until placements resume
inline size_t next_batch_size(size_t bsz, size_t bmax, bool failed) {
    return failed ? std::max<size_t>(std::min<size_t>(64, bmax), bsz / 4) : std::min<size_t>(bmax, bsz * 2);
}

constexpr const char* GANG_TOO_BIG = "yk_cycle: a gang has more members than the sweep batch (raise yk_config.batch)";

// Fills the next batch: at most bsz asks, at most cap_user of them.  A gang larger than bsz raises bsz to bmax; false when
// not even bmax holds it.
inline bool fill_batch(Orderer& ord, size_t& bsz, size_t bmax, size_t cap_user, std::vector<uint32_t>& asks, Orderer::Snap& snap,
                       yk_stats_t& st) {
    asks.clear();
    if (cap_user == 0) return true;
    const auto t0 = std::chrono::steady_clock::now();
    ord.fill(bsz, cap_user, asks, snap);
    if (ord.oversize_gang && bsz < bmax) { bsz = bmax; ord.fill(bsz, cap_user, asks, snap); }
    st.host_ms[2] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return !ord.oversize_gang;
}

inline bool same_gang(const Tables& t, uint32_t x, uint32_t y) {
    return t.a_gang[x] != CNONE && t.a_gang[x] == t.a_gang[y] && t.a_app[x] == t.a_app[y];
}

// Decided entries [0, consumed) of a batch: orderer bookkeeping, and bind(ask, node) for every placement.  Returns whether
// the batch ended on an ask / gang that found no node in a placement-sensitive order: the orderer is then rewound to just
// before it (`later`, a batch filled after this one, is undone as well).
template <class Bind>
inline bool settle(Orderer& ord, const std::vector<uint32_t>& asks, Orderer::Snap& snap, Orderer::Snap* later, const uint32_t* result,
                   size_t consumed, bool ins, yk_stats_t& st, Bind&& bind) {
    bool failed = false;
    if (!ins && consumed > 0 && result[consumed - 1] == CNONE) {
        const auto t0 = std::chrono::steady_clock::now();
        size_t j = consumed - 1;   // first entry of the failed ask / gang
        while (j > 0 && same_gang(ord.t, asks[j], asks[j - 1]) && result[j - 1] == CNONE) --j;
        ord.rewind(snap, later, asks, j);
        st.host_ms[2] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        failed = true;
    }
    for (size_t i = 0; i < consumed; ++i) {
        const uint32_t a = asks[i];
        if (result[i] == CNONE) {
            if (ins) ord.fail_in_place(a);
            st.nofit++;
            continue;
        }
        ord.confirm(a);
        bind(a, result[i]);
        st.allocations++;
    }
    return failed;
}

}  // namespace yk

namespace ykun {

constexpr size_t UN_EMAX = (size_t)4 << 20;   // generated elements per attempt at most (nodes x depth)

// The attempts of one uniform run of R asks requesting `req`, on the live nodes `live` (totals column-major, leading
// dimension ldn).  attempt(L, g) runs one attempt at depth L and leaves its Globals in g; a non-zero return is an error and
// is passed on.  Afterwards *status is U_DONE / U_STOPPED with *consumed entries decided, U_FALLBACK (nothing was applied:
// the windowed commit takes the run) or U_NAN (a node scores NaN after the commit).  Under binpacking an attempt is one
// ordered capacity fill (yk_uniform.h), made once: attempt(1, g).
template <class Attempt>
inline int uniform_run(int D, const double* w, const int64_t* req, const int64_t* n_total, size_t ldn, const uint32_t* live, int nlive,
                       int R, int first_override, yk_stats_t& st, Attempt&& attempt, int* status, size_t* consumed,
                       bool binpacking = false) {
    *status = U_FALLBACK; *consumed = 0;
    if (nlive == 0 || R == 0) return 0;
    if (binpacking) {
        if ((size_t)nlive > UN_EMAX) return 0;   // the keys do not fit the element buffers: fallback
        Globals g{};
        const int rc = attempt(1, g);
        if (rc) return rc;
        if (g.status == U_FALLBACK) return 0;
        if (g.status == U_NAN || g.nan) { *status = U_NAN; return 0; }
        *status = g.status; *consumed = (size_t)g.consumed;
        st.uniform_runs++; st.uniform_asks += (uint64_t)g.consumed; st.uniform_elements += (uint64_t)nlive;
        return 0;
    }
    int L = first_depth(R, nlive);
    // no node takes the request more often than its TOTAL allows: beyond that depth nothing is ever cut
    int64_t capmax = 0;
    for (int i = 0; i < nlive; ++i) {
        int64_t tot[8];
        for (int k = 0; k < D; ++k) tot[k] = n_total[(size_t)k * ldn + live[i]];
        capmax = std::max(capmax, cap_of_d(D, true, tot, tot, req, (int64_t)R));
    }
    int Lmax = 1;
    while ((int64_t)Lmax < capmax) Lmax <<= 1;
    {   // a request with no weighted dimension leaves every key where it is: the run fills the first nodes (by key, NodeID) to
        // the brim, so the depth that matters is a node's whole capacity, not the mean share
        bool flat = true;
        for (int k = 0; k < D; ++k) if (w[k] != 0.0 && req[k] != 0) flat = false;
        if (flat) L = Lmax;
    }
    if (first_override > 0) L = first_override;   // testing knob: a shallow first attempt makes the retry path reachable
    L = std::min(L, Lmax);
    for (;;) {
        if ((size_t)L * (size_t)nlive > UN_EMAX) return 0;   // too deep for the element buffers: fallback
        Globals g{};
        const int rc = attempt(L, g);
        if (rc) return rc;
        if (g.status == U_RETRY) {   // deeper; past Lmax only if a node's available exceeds its total (the buffers end it)
            st.uniform_retries++;
            L = L < Lmax ? (int)std::min<int64_t>((int64_t)L * 4, (int64_t)Lmax) : L * 4;
            continue;
        }
        if (g.status == U_NAN || g.status == U_FALLBACK) return 0;
        if (g.nan) { *status = U_NAN; return 0; }
        *status = g.status; *consumed = (size_t)g.consumed;
        st.uniform_runs++; st.uniform_asks += (uint64_t)g.consumed; st.uniform_elements += (uint64_t)L * (uint64_t)nlive;
        return 0;
    }
}

}  // namespace ykun

namespace yklt {

inline bool same_request(const yk::CommitTables& t, uint32_t a, uint32_t b) {
    for (int k = 0; k < t.D; ++k)
        if (t.a_req[(size_t)k * t.lda + a] != t.a_req[(size_t)k * t.lda + b]) return false;
    return true;
}

// Dense numbers for the distinct request vectors ("shapes") of the cycle's pending asks: a_shape[ask].  Equal numbers <=>
// equal vectors (hash table, equality always confirmed on the full vector).
inline void assign_shapes(const yk::CommitTables& t, const std::vector<uint32_t>& pending, std::vector<uint32_t>& a_shape, uint32_t* n_shapes) {
    struct Slot { uint32_t ask; uint32_t id; };
    size_t cap = 64;
    while (cap < 4 * pending.size()) cap <<= 1;
    std::vector<Slot> shapes(cap, Slot{yk::CNONE, 0});
    uint32_t ns = 0;
    for (uint32_t a : pending) {
        uint64_t h = 0x9E3779B97F4A7C15ull;
        for (int k = 0; k < t.D; ++k) { h ^= (uint64_t)t.a_req[(size_t)k * t.lda + a] + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); h *= 0xD6E8FEB86659FD93ull; }
        size_t x = (size_t)(h ^ (h >> 29)) & (cap - 1);
        for (;;) {
            Slot& s = shapes[x];
            if (s.ask == yk::CNONE) { s.ask = a; s.id = ns++; a_shape[a] = s.id; break; }
            if (same_request(t, s.ask, a)) { a_shape[a] = s.id; break; }
            x = (x + 1) & (cap - 1);
        }
    }
    *n_shapes = ns;
}

// Dense numbers for the distinct predicate signatures of the given asks (the engine keeps these up to date as asks are
// upserted; the CPU test harness computes them here).  a_sig = the 64-bit signature hashes.
inline void assign_sigs(const yk::CommitTables& t, const uint64_t* a_sig, const std::vector<uint32_t>& pending, std::vector<uint32_t>& a_sigid) {
    struct Slot { uint32_t ask; uint32_t id; };
    size_t cap = 64;
    while (cap < 4 * pending.size()) cap <<= 1;
    std::vector<Slot> sigs(cap, Slot{yk::CNONE, 0});
    uint32_t ng = 0;
    for (uint32_t a : pending) {
        const uint64_t g = a_sig[a];
        size_t x = (size_t)(g ^ (g >> 29)) & (cap - 1);
        for (;;) {
            Slot& s = sigs[x];
            if (s.ask == yk::CNONE) { s.ask = a; s.id = ng++; a_sigid[a] = s.id; break; }
            if (a_sig[s.ask] == g && yk::same_signature(t, s.ask, a)) { a_sigid[a] = s.id; break; }
            x = (x + 1) & (cap - 1);
        }
    }
}

// the three words per batch entry that the kernel reads (yk_lattice.h): gang flags, shape number, signature number
inline void build_meta(const yk::CommitTables& t, const uint32_t* a_shape, const uint32_t* a_sigid, const std::vector<uint32_t>& batch,
                       uint32_t* meta, uint32_t* shp, uint32_t* sig) {
    const size_t B = batch.size();
    for (size_t i = 0; i < B; ++i) {
        const uint32_t a = batch[i];
        uint32_t m = 0;
        if (t.a_gang[a] != yk::CNONE) {
            m |= M_GANG;
            const uint32_t b = i ? batch[i - 1] : a;
            if (i == 0 || t.a_gang[b] != t.a_gang[a] || t.a_app[b] != t.a_app[a]) m |= M_GSTART;
        }
        meta[i] = m; shp[i] = a_shape[a]; sig[i] = a_sigid[a];
    }
}

// How many sub-run windows the kernel's staging rules (at most SMAX shapes, SIGCAP signatures, KCAP asks) cut the batch
// into at least: the engine only starts a cycle on the device commit when the windows are long enough to pay for a sub-run.
inline size_t estimate_windows(const uint32_t* shp, const uint32_t* sig, size_t B) {
    size_t windows = 0, i = 0;
    std::vector<uint32_t> seen(512, 0xFFFFFFFFu);
    while (i < B) {
        uint32_t shapes[SMAX];
        int ns = 0, rows = 0;
        std::fill(seen.begin(), seen.end(), 0xFFFFFFFFu);
        size_t j = i;
        for (; j < B && j - i < (size_t)KCAP; ++j) {
            int k = 0;
            while (k < ns && shapes[k] != shp[j]) ++k;
            if (k == ns) { if (ns == SMAX) break; shapes[ns++] = shp[j]; }
            size_t x = (sig[j] * 2654435761u) >> 23;   // 9 bits
            while (seen[x] != 0xFFFFFFFFu && seen[x] != sig[j]) x = (x + 1) & 511;
            if (seen[x] == 0xFFFFFFFFu) { if (rows == SIGCAP) break; seen[x] = sig[j]; ++rows; }
        }
        ++windows;
        i = j > i ? j : i + 1;
    }
    return windows;
}

// What the lattice commit relies on (DESIGN.md "lattice commit"):
//   fair node sort; weights >= 0 and weighted totals >= 0 (a node's key must not decrease when it is allocated to; under
//   binpacking, which a caller may allow for the binpacking fill, it must not increase);
//   NodeID ranks unique (element order is (key, rank, j)); every gang's members request the same vector (a gang never
//   straddles two runs, so a failed gang is undone inside one sub-run).
struct Eligibility {
    bool ok = false;
    const char* why = "";
};

// ranks_unique: when the caller already knows whether the live nodes' ranks are distinct (the engine checks it where it sorts
// the nodes by rank), else nullptr; any_gang: when it already knows whether any pending ask is a gang member; binpacking_ok:
// the binpacking node sort is accepted (YK_FLAG_BINPACKING_DEVICE).
inline Eligibility eligible(const yk::CommitTables& t, uint32_t n_hi, const uint8_t* n_present, const int64_t* n_total,
                            size_t ldn, const uint32_t* n_rank, const std::vector<uint32_t>& pending, const bool* ranks_unique = nullptr,
                            const bool* any_gang = nullptr, bool binpacking_ok = false) {
    Eligibility e;
    if (t.policy != 0u && !(t.policy == 1u && binpacking_ok)) { e.why = "binpacking node sort"; return e; }
    for (int k = 0; k < t.D; ++k) if (t.w[k] < 0.0 || t.w[k] != t.w[k]) { e.why = "negative node-sort weight"; return e; }
    for (int k = 0; k < t.D; ++k) {
        if (t.w[k] == 0.0) continue;
        const int64_t* col = n_total + (size_t)k * ldn;
        for (uint32_t n = 0; n < n_hi; ++n)
            if (n_present[n] && col[n] < 0) { e.why = "negative total on a weighted resource"; return e; }
    }
    if (ranks_unique) {
        if (!*ranks_unique) { e.why = "duplicate NodeID ranks"; return e; }
    } else {
        std::vector<uint32_t> ranks;
        ranks.reserve(n_hi);
        for (uint32_t n = 0; n < n_hi; ++n) if (n_present[n]) ranks.push_back(n_rank[n]);
        std::sort(ranks.begin(), ranks.end());
        for (size_t i = 1; i < ranks.size(); ++i) if (ranks[i] == ranks[i - 1]) { e.why = "duplicate NodeID ranks"; return e; }
    }
    if (!any_gang || *any_gang) {
        std::unordered_map<uint64_t, uint32_t> first;   // (app, gang) -> first member seen
        for (uint32_t a : pending) {
            if (t.a_gang[a] == yk::CNONE) continue;
            const uint64_t key = ((uint64_t)t.a_app[a] << 32) | t.a_gang[a];
            auto it = first.find(key);
            if (it == first.end()) first.emplace(key, a);
            else if (!same_request(t, a, it->second)) { e.why = "a gang mixes request vectors"; return e; }
        }
    }
    e.ok = true;
    return e;
}

// One planned batch (ykun::plan_segments): uniform runs through uniform(off, len, has_gang, &ykun_status, &consumed), which
// hands a run it cannot decide to the window with U_FALLBACK, the stretches between them through window(off, len, &status,
// &consumed).  *status and *consumed describe the whole batch: the first segment that does not finish ends it.
template <class Uniform, class Window>
inline int run_segments(const std::vector<ykun::Segment>& segs, const uint32_t* meta, Uniform&& uniform, Window&& window,
                        int* status, size_t* consumed) {
    *status = ST_DONE; *consumed = 0;
    for (const ykun::Segment& sg : segs) {
        size_t cons = 0;
        int st = ST_DONE;
        bool windowed = !sg.uniform;
        if (sg.uniform) {
            bool has_gang = false;
            for (int i = 0; i < sg.len && !has_gang; ++i) has_gang = (meta[(size_t)sg.off + i] & M_GANG) != 0;
            int ust = ykun::U_FALLBACK;
            const int rc = uniform((size_t)sg.off, (size_t)sg.len, has_gang, &ust, &cons);
            if (rc) return rc;
            if (ust == ykun::U_FALLBACK) windowed = true;
            else st = ust == ykun::U_NAN ? ST_NAN : ust == ykun::U_STOPPED ? ST_STOPPED : ST_DONE;
        }
        if (windowed) {
            const int rc = window((size_t)sg.off, (size_t)sg.len, &st, &cons);
            if (rc) return rc;
        }
        *consumed = (size_t)sg.off + cons;
        *status = st;
        if (st != ST_DONE || cons < (size_t)sg.len) break;
    }
    return 0;
}

// The window callback of run_segments under binpacking, where a batch is planned with min_run = 1 (every segment a maximal
// uniform run, each decided by one fill): a segment the fill cannot decide -- a run whose gang may need a roll-back
// (U_FALLBACK), or a stretch cut inside a gang whose members carry different signatures -- and everything after it goes to
// the host commit.
inline int hand_off(size_t, size_t, int* status, size_t* consumed) {
    *status = ST_HANDOFF; *consumed = 0;
    return 0;
}

// Whether the round commit (yk_rounds.h) may decide a stretch of asks: a placement-insensitive order (a NOFIT fails in
// place), no gang member, and no masks -- no required or forbidden labels, no node name, every taint of the live nodes
// (`taints`, their union) tolerated.
inline bool round_eligible(const yk::CommitTables& t, bool insensitive, uint64_t taints, const uint32_t* asks, size_t len) {
    if (!insensitive) return false;
    for (size_t i = 0; i < len; ++i) {
        const uint32_t a = asks[i];
        if (t.a_gang[a] != yk::CNONE || t.a_need[a] || t.a_deny[a] || t.a_node[a] != yk::CNONE || (taints & ~t.a_tol[a])) return false;
    }
    return true;
}

// The window callback of run_segments for a cycle on the device commit: a round-eligible stretch goes through
// rounds(off, len, &status, &consumed) when `rounds_on`, every other one through window(...).
template <class Rounds, class Window>
inline auto route_stretches(bool rounds_on, const yk::CommitTables& t, bool insensitive, uint64_t taints, const uint32_t* asks,
                            Rounds& rounds, Window& window) {
    return [=, &t, &rounds, &window](size_t off, size_t len, int* status, size_t* consumed) -> int {
        if (rounds_on && round_eligible(t, insensitive, taints, asks + off, len)) return rounds(off, len, status, consumed);
        return window(off, len, status, consumed);
    };
}

// What the device commit's batch loop works on; the caller owns all of it.
struct Loop {
    yk::Orderer& ord;
    const yk::CommitTables& ct;
    const uint32_t* shape_ids; const uint32_t* sig_ids;   // build_meta's numbers per ask
    std::vector<uint32_t>& asks; yk::Orderer::Snap& snap;   // the batch being decided (the first one already filled)
    std::vector<uint32_t>& result;                          // its node per entry, NONE for none
    uint32_t* meta; uint32_t* shp; uint32_t* sig;           // its per-entry words
    std::vector<ykun::Segment>& segs;
    bool& plan_ready;                                       // meta and segs already describe the first batch
    int min_run;                                            // shortest uniform run (0: none)
    bool no_nodes;
    size_t bmax;                                            // largest batch
    uint32_t max_bindings; const uint32_t& n;               // bindings allowed in the cycle, made so far
    yk_stats_t& st;
};

// The cycle on the device commit, batch by batch.  batch(B, &status, &consumed) decides one batch into lp.result[0,
// consumed); bind(ask, node) takes a binding (and counts it in lp.n); fail(yk_status, message) reports an error.  Returns
// with handoff = true, lp.asks holding the decided prefix only, when a gang has to be rolled back after a partial
// placement: the rest of the cycle belongs to the host commit.
template <class Batch, class Bind, class Fail>
inline int device_commit(Loop& lp, Batch&& batch, Bind&& bind, Fail&& fail, bool& handoff) {
    handoff = false;
    const bool ins = lp.ord.insensitive;
    size_t bsz = lp.bmax;
    while (!lp.asks.empty()) {
        const size_t B = lp.asks.size();
        if (!lp.plan_ready) {
            build_meta(lp.ct, lp.shape_ids, lp.sig_ids, lp.asks, lp.meta, lp.shp, lp.sig);
            ykun::plan_segments(lp.meta, lp.shp, lp.sig, (int)B, lp.min_run > 0 ? lp.min_run : (int)B + 1, lp.segs);
        }
        lp.plan_ready = false;
        size_t consumed = 0;
        int status = ST_DONE;
        if (lp.no_nodes) {   // nothing fits
            lp.result.assign(B, NONE);
            consumed = ins ? B : 1;
            if (!ins) status = ST_STOPPED;
            while (!ins && consumed < B && yk::same_gang(lp.ord.t, lp.asks[0], lp.asks[consumed])) ++consumed;
        } else {
            const int rc = batch(B, &status, &consumed);
            if (rc) return rc;
            if (status == ST_NAN) return fail(YK_ERR_RANGE, "NaN node score after commit");
        }
        lp.st.lattice_asks += consumed;
        lp.st.batches++;
        if (status == ST_HANDOFF) {
            lp.ord.unfill(lp.snap, lp.asks, consumed);   // the undecided tail goes back to the orderer
            lp.asks.resize(consumed);
            lp.result.resize(consumed);
            // no failure cut: every decided entry stands (a placement-sensitive batch never carries a NONE before a hand-over,
            // the kernel stops there instead; an insensitive one fails NONE entries in place)
            yk::settle(lp.ord, lp.asks, lp.snap, nullptr, lp.result.data(), consumed, true, lp.st, bind);
            lp.st.lattice_handoffs++;
            handoff = true;
            return 0;
        }
        const bool failed = yk::settle(lp.ord, lp.asks, lp.snap, nullptr, lp.result.data(), consumed, ins, lp.st, bind);
        if (!failed && consumed < B) return fail(YK_ERR_CUDA, "lattice kernel ended a batch early without a failure");
        bsz = yk::next_batch_size(bsz, lp.bmax, failed);
        if (!yk::fill_batch(lp.ord, bsz, lp.bmax, (size_t)lp.max_bindings - lp.n, lp.asks, lp.snap, lp.st)) return fail(YK_ERR_ARG, yk::GANG_TOO_BIG);
    }
    return 0;
}

}  // namespace yklt
