// yk_commit.hpp -- the ordered commit: turns the fit bitmaps of a batch into bindings that are identical to what the
// reference's one-allocation-per-pass loop would produce (DESIGN.md "ordered commit").  Host code, no CUDA: both the
// engine (yk_engine.cu) and tests/host/engine_shim.cpp run it under one batch loop, yk::host_commit (yk_lattice_host.hpp);
// the engine feeds it rows as they arrive from the device, the shim rows computed on the CPU, so that this logic --
// epochs, the touched-node index, gang roll-back -- and the loop around it are exercised by the CPU test suite.
//
// Invariant it relies on: within an epoch a node that has not been committed to still has exactly the state the sorted
// view (and therefore the bitmaps) was built from.  For ask i:
//   (A) best untouched candidate = first set bit of fit[i] & ~touched, in sorted (score, NodeID) order;
//   (B) best touched candidate   = first entry of the touched-node index (ordered by CURRENT (score, NodeID)) that sorts
//       before (A) and passes the full predicate on the working copy;
//   the ask takes (B) if it exists, else (A); the node's availability drops, it is re-scored and re-indexed.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>
#if defined(__x86_64__)
#include <x86intrin.h>
#endif

#include "yk_dirty.hpp"
#include "yk_score.h"

namespace yk {

constexpr uint32_t CNONE = 0xFFFFFFFFu;
constexpr int CMAX_D = 8;

// views of the engine's host tables that the commit reads
struct CommitTables {
    int D = 0;
    uint32_t policy = 0;
    const double* w = nullptr;       // [D] node-sort weights
    size_t lda = 0;                  // ask tables are column-major with this stride
    const int64_t* a_req = nullptr;  // [D][lda]
    const uint64_t* a_tol = nullptr;
    const uint64_t* a_need = nullptr;
    const uint64_t* a_deny = nullptr;
    const uint32_t* a_node = nullptr;
    const uint32_t* a_gang = nullptr;
    const uint32_t* a_app = nullptr;
};

// ---- shared rows ----------------------------------------------------------------------------------------------
// What the sweep computes for an ask depends only on (request, tolerations, required / forbidden labels, node name):
// asks of one deployment / job / task group are identical there.  The batch is therefore swept once per DISTINCT
// signature: rows[] lists one representative ask per signature (in order of first appearance, so rows land in the
// order the commit first needs them) and row_of[i] is the row of batch entry i.  The 64-bit signature hash is
// computed once when an ask is upserted; equality is always confirmed on the full signature.
inline uint64_t ask_signature(const CommitTables& t, uint32_t a) {
    // every field gets its own odd multiplier (independent multiplies: no serial chain), folded by xor / rotate, one
    // final avalanche.  Collisions only cost a full compare: equality is never decided on the hash.
    static const uint64_t C[12] = {0x9E3779B97F4A7C15ull, 0xC2B2AE3D27D4EB4Full, 0x165667B19E3779F9ull, 0xD6E8FEB86659FD93ull,
                                   0xFF51AFD7ED558CCDull, 0xC4CEB9FE1A85EC53ull, 0x2545F4914F6CDD1Dull, 0x94D049BB133111EBull,
                                   0xBF58476D1CE4E5B9ull, 0xA0761D6478BD642Full, 0xE7037ED1A0B428DBull, 0x8EBC6AF09C88C6E3ull};
    uint64_t h = 0x243F6A8885A308D3ull;
    for (int k = 0; k < t.D; ++k) {
        const uint64_t v = (uint64_t)t.a_req[(size_t)k * t.lda + a] * C[k];
        h ^= (v << (7 * k + 1)) | (v >> (63 - 7 * k));
    }
    h ^= t.a_tol[a] * C[8];
    h ^= (t.a_need[a] * C[9]) >> 3 | (t.a_need[a] * C[9]) << 61;
    h ^= (t.a_deny[a] * C[10]) >> 17 | (t.a_deny[a] * C[10]) << 47;
    h ^= ((uint64_t)t.a_node[a] + 1) * C[11];
    h ^= h >> 32;
    h *= 0xD6E8FEB86659FD93ull;
    return h ^ (h >> 29);
}
inline bool same_signature(const CommitTables& t, uint32_t a, uint32_t b) {
    if (t.a_tol[a] != t.a_tol[b] || t.a_need[a] != t.a_need[b] || t.a_deny[a] != t.a_deny[b] || t.a_node[a] != t.a_node[b]) return false;
    for (int k = 0; k < t.D; ++k)
        if (t.a_req[(size_t)k * t.lda + a] != t.a_req[(size_t)k * t.lda + b]) return false;
    return true;
}

class RowShare {
public:
    // share == false: one row per ask (rows = batch, row_of = identity)
    void build(const CommitTables& t, const uint64_t* a_sig, const std::vector<uint32_t>& batch, bool share,
               std::vector<uint32_t>& rows, std::vector<uint32_t>& row_of) {
        const size_t B = batch.size();
        rows.clear();
        row_of.resize(B);
        if (!share) {
            rows = batch;
            for (size_t i = 0; i < B; ++i) row_of[i] = (uint32_t)i;
            return;
        }
        size_t cap = 64;
        while (cap < 2 * B) cap <<= 1;
        if (slot_.size() < cap) { slot_.assign(cap, Entry{0, 0, 0}); stamp_ = 0; }
        if (++stamp_ == 0) { std::fill(slot_.begin(), slot_.end(), Entry{0, 0, 0}); stamp_ = 1; }
        const size_t mask = slot_.size() - 1;
        for (size_t i = 0; i < B; ++i) {
            const uint32_t a = batch[i];
            const uint64_t h = a_sig[a];
            size_t x = (size_t)(h ^ (h >> 29)) & mask;
            while (true) {
                Entry& e = slot_[x];
                if (e.stamp != stamp_) {   // free in this batch: a new signature
                    e.stamp = stamp_; e.sig = h; e.row = (uint32_t)rows.size();
                    row_of[i] = e.row;
                    rows.push_back(a);
                    break;
                }
                if (e.sig == h && same_signature(t, rows[e.row], a)) { row_of[i] = e.row; break; }
                x = (x + 1) & mask;
            }
        }
    }

private:
    struct Entry { uint64_t sig; uint32_t row; uint32_t stamp; };
    std::vector<Entry> slot_;
    uint32_t stamp_ = 0;
};

// The per-node working record lives in one contiguous slice of `hot` (hs = 4 + 3D words):
//   [0] sort key (valid while the node is touched)   [1] rank<<32 | touched<<31 | retired<<30   [2] taint   [3] label
//   [4,4+D) cap = min(max(0,total), max(0,available))   -- first 64 bytes at D = 4: all a predicate re-check touches
//   [4+D,4+2D) available   [4+2D,4+3D) total            -- only read when the node is actually committed to
struct NodeView {
    int64_t* h; int D;
    uint64_t& key() { return *reinterpret_cast<uint64_t*>(&h[0]); }
    uint32_t rank() const { return (uint32_t)((uint64_t)h[1] >> 32); }
    bool dirty() const { return (((uint64_t)h[1]) >> 31) & 1u; }
    void set_rank(uint32_t rank) { h[1] = (int64_t)((uint64_t)rank << 32); }   // also clears the touched flag
    bool retired() const { return (((uint64_t)h[1]) >> 30) & 1u; }
    void set_dirty(bool d) { h[1] = (int64_t)((((uint64_t)h[1]) & ~0xC0000000ull) | (d ? 0x80000000ull : 0ull)); }   // clears `retired` too
    void set_retired(bool r) { h[1] = (int64_t)((((uint64_t)h[1]) & ~0x40000000ull) | (r ? 0x40000000ull : 0ull)); }
    int64_t* cap() { return h + 4; }
    int64_t* avail() { return h + 4 + D; }
    int64_t* total() { return h + 4 + 2 * D; }
    void recap() {   // after `available` changed
        for (int k = 0; k < D; ++k) {
            const int64_t a = avail()[k] < 0 ? 0 : avail()[k], t = total()[k] < 0 ? 0 : total()[k];
            cap()[k] = a < t ? a : t;
        }
    }
};

inline unsigned long long commit_tsc() {
#if defined(__x86_64__)
    unsigned aux;
    unsigned long long t = __rdtscp(&aux);
    _mm_lfence();
    return t;
#else
    return 0;
#endif
}

class Committer {
public:
    CommitTables t;
    std::vector<int64_t> hot;            // working copy of the node table (see NodeView)
    int hs = 0;
    DirtyIndex dirty;                    // nodes touched in this epoch, ordered by their CURRENT (score, NodeID)
    std::vector<DirtyRef> dirty_sorted;  // scratch for the epoch-end merge
    std::vector<uint32_t> dirty_words;   // bit p = the node at sorted position p has been touched in this epoch
    std::vector<uint32_t> dirty_list;    // the touched nodes, in first-touch order
    // Touched nodes that can no longer hold ANY pending ask of the cycle (some dimension is below the smallest request
    // of the cycle in that dimension) are retired: kept out of the walked index -- a binpacking cycle would otherwise
    // step over every node it has filled, for every ask -- and put back into the order at the epoch end.
    std::vector<DirtyRef> retired_refs;
    int64_t cycle_min_req[CMAX_D];       // per dimension: smallest request among the cycle's pending asks
    std::vector<DirtyRef> oref[2];       // node order of the epoch: sorted position -> (key, rank, node); double-buffered
    int ocur = 0;
    int64_t dirty_ub[CMAX_D];            // per dimension: upper bound of cap over the touched nodes
    // Per row of the current batch: a frontier in the touched order below which no entry fits that row's signature.
    // Within an epoch a touched node only loses availability, so "does not fit signature r" is permanent, except for the
    // nodes a gang roll-back hands back: walks for r start at the frontier instead of the front, after replaying from
    // ins_log the entries (re)inserted -- by commits and by roll-backs -- since the row last looked.  Without this, a
    // binpacking cycle walks over every node it has already filled, for every ask.
    struct RowSkip { DirtyRef skip; uint32_t seen; };
    std::vector<RowSkip> rskip;
    std::vector<uint32_t> ins_log;       // nodes (re)inserted into the touched order during this batch
    bool skip_active = false;
    int front = 0;                       // every sorted position below word `front` is touched
    int W = 0;                           // bitmap words per row in this epoch
    bool profile = false;
    uint64_t dbg[4] = {0, 0, 0, 0};      // words scanned, touched candidates examined, asks won by a touched node, re-keys
    uint64_t prof[6] = {0, 0, 0, 0, 0, 0};

    NodeView node(uint32_t n) { return NodeView{hot.data() + (size_t)n * hs, t.D}; }

    // (re)build the working copy from the engine's column-major host tables (stride ldn), n_hi node slots
    void build(uint32_t n_hi, const int64_t* n_avail, const int64_t* n_total, size_t ldn, const uint64_t* n_taint,
               const uint64_t* n_label, const uint32_t* n_rank) {
        const int D = t.D;
        hs = 4 + 3 * D;
        hot.resize((size_t)n_hi * hs);
        for (int k = 0; k < D; ++k) {   // index order: sequential reads of the column-major tables
            const int64_t* av = n_avail + (size_t)k * ldn;
            const int64_t* to = n_total + (size_t)k * ldn;
            int64_t* h = hot.data();
            for (uint32_t n = 0; n < n_hi; ++n) { h[(size_t)n * hs + 4 + D + k] = av[n]; h[(size_t)n * hs + 4 + 2 * D + k] = to[n]; }
        }
        for (uint32_t n = 0; n < n_hi; ++n) {
            NodeView v = node(n);
            v.h[0] = 0;
            v.set_rank(n_rank[n]);
            v.h[2] = (int64_t)n_taint[n];
            v.h[3] = (int64_t)n_label[n];
            v.recap();
        }
    }

    // the cycle's initial node order (ascending (score key, NodeID rank)), as the device sort produced it
    void set_order(const uint32_t* nodes, const uint64_t* keys, int nlive) {
        ocur = 0;
        oref[0].resize((size_t)nlive);
        oref[1].resize((size_t)nlive);
        for (int p = 0; p < nlive; ++p) oref[0][(size_t)p] = DirtyRef(keys[p], node(nodes[p]).rank(), nodes[p]);
    }
    const DirtyRef* order() const { return oref[ocur].data(); }

    // once per cycle, before the first batch: what the smallest pending request is in every dimension
    void set_pending(const std::vector<uint32_t>& pending) {
        for (int k = 0; k < CMAX_D; ++k) cycle_min_req[k] = INT64_MIN;   // nothing is ever below it: retire nothing
        if (pending.empty()) return;
        for (int k = 0; k < t.D; ++k) {
            const int64_t* col = t.a_req + (size_t)k * t.lda;
            int64_t m = INT64_MAX;
            for (uint32_t a : pending) m = std::min(m, col[a]);
            cycle_min_req[k] = m;
        }
    }

    // a new epoch starts on a fresh view of `words` bitmap words per row: nothing is touched
    void begin_epoch(int words) {
        retired_refs.clear();
        for (uint32_t n : dirty_list) node(n).set_dirty(false);
        dirty_list.clear();
        dirty.clear();
        front = 0;
        W = words;
        dirty_words.assign((size_t)words, 0);
        for (int k = 0; k < CMAX_D; ++k) dirty_ub[k] = INT64_MIN;
    }

    // full (ask,node) predicate on the working copy, for touched nodes (they were chosen before: schedulable, unreserved).
    // Same steps as the sweep kernel; everything it reads sits in the first 64 bytes of the record at D = 4.
    bool fits_now(uint32_t n, uint32_t ask) const {
        const int64_t* h = hot.data() + (size_t)n * hs;
        const uint64_t taint = (uint64_t)h[2], label = (uint64_t)h[3];
        if ((taint & ~t.a_tol[ask]) | (~label & t.a_need[ask]) | (label & t.a_deny[ask])) return false;
        if (t.a_node[ask] != CNONE && t.a_node[ask] != n) return false;
        for (int k = 0; k < t.D; ++k)
            if (t.a_req[(size_t)k * t.lda + ask] > h[4 + k]) return false;
        return true;
    }

    bool same_gang(uint32_t x, uint32_t y) const {
        return t.a_gang[x] != CNONE && t.a_gang[x] == t.a_gang[y] && t.a_app[x] == t.a_app[y];
    }

    // Ordered commit of one batch.  fit = rows of WS = W+1 words (W bitmap words, then the first-fit position);
    // row_of[i] = the row of batch entry i (see RowShare); wait(r) blocks
    // until row r has landed and returns how many rows have (>= r+1), or a negative status.  result[i] = node or CNONE; consumed = entries decided (the loop stops
    // after the first failed ask / gang unless the order is placement-insensitive).  Returns 0, or wait()'s error,
    // or -5 when a re-score is NaN.
    template <typename WaitFn>
    int commit_batch(const std::vector<uint32_t>& batch, const uint32_t* row_of, const uint32_t* fit,
                     bool insensitive, std::vector<uint32_t>& result, size_t& consumed, WaitFn&& wait) {
        const DirtyRef* order = oref[ocur].data();
        const int D = t.D;
        const int B = (int)batch.size();
        const int WS = W + 1;
        result.assign((size_t)B, CNONE);
        consumed = 0;
        {
            uint32_t nrows = 0;
            for (int i = 0; i < B; ++i) nrows = std::max(nrows, row_of[(size_t)i] + 1);
            rskip.assign(nrows, RowSkip{DirtyRef(), 0});
            ins_log.clear();
            skip_active = false;
        }
        int landed = 0;
        bool stop = false;
        // all-or-nothing gangs: commits of the gang in progress are logged so they can be undone
        struct Undo { uint32_t node; uint32_t pos; uint64_t old_key; bool was_dirty; int64_t old_avail[CMAX_D]; };
        std::vector<Undo> undo;
        int gang_begin = -1;
        for (int i = 0; i < B && !stop; ++i) {
            const int ri = (int)row_of[(size_t)i];
            if (ri >= landed) {
                const int rc = wait(ri);
                if (rc < 0) return rc;
                landed = rc;
            }
            const unsigned long long tc0 = profile ? commit_tsc() : 0;
            const uint32_t ask = batch[(size_t)i];
            const bool in_gang = t.a_gang[ask] != CNONE;
            if (in_gang && (i == 0 || !same_gang(batch[(size_t)i - 1], ask))) { gang_begin = i; undo.clear(); }
            const uint32_t* row = fit + (size_t)ri * WS;
            if (i + 12 < B && (int)row_of[(size_t)i + 12] < landed) {   // rows arrive by DMA and are cache-cold: pull
                const uint32_t* nrow = fit + (size_t)row_of[(size_t)i + 12] * WS;   // the first-fit word of a landed row now
                __builtin_prefetch(nrow + W);                        // ... and, for the row whose first-fit word was
                const uint32_t* mrow = fit + (size_t)row_of[(size_t)i + 6] * WS;   // pulled six asks ago, the line its scan starts at
                const uint32_t nf = mrow[W];
                __builtin_prefetch(mrow + std::min<int>(W, std::max<int>(front, nf == CNONE ? 0 : (int)(nf >> 5))));
            }
            // (A) best untouched node: first set bit of row & ~touched in sorted order
            uint32_t posA = CNONE;
            const uint32_t f = row[W];
            if (f != CNONE) {
                while (front < W && dirty_words[(size_t)front] == 0xFFFFFFFFu) ++front;
                for (int wd = std::max((int)(f >> 5), front); wd < W; ++wd) {
                    ++dbg[0];
                    const uint32_t m = row[wd] & ~dirty_words[(size_t)wd];
                    if (m) { posA = (uint32_t)wd * 32u + (uint32_t)__builtin_ctz(m); break; }
                }
            }
            DirtyRef bound(~0ull, ~0u, CNONE);
            if (posA != CNONE) {
                bound = order[posA];
                // the clean candidate wins about half the time; on big clusters its record is not in cache: start
                // pulling both lines now, the walk below hides the latency
                const int64_t* rec = hot.data() + (size_t)bound.node() * hs;
                __builtin_prefetch(rec);
                __builtin_prefetch(rec + 8);
            }
            const unsigned long long tc1 = profile ? commit_tsc() : 0;
            // (B) best re-scored node among those touched earlier in this epoch.  dirty_ub prunes the walk: if the
            // request exceeds what ANY touched node has left on some dimension, none of them can fit.  A walk that ran
            // over the whole index without a fit leaves the bound exact (it saw every touched node), which keeps a full
            // cluster cheap: the first failing ask pays for the walk, the following ones are pruned.
            uint32_t chosen = CNONE;
            DirtyIndex::Cursor cur;
            bool at_cursor = false;   // `chosen` is the entry the cursor stands on (taken out without a search)
            bool may_fit = f != CNONE && dirty.size() > 0;
            if (may_fit)
                for (int k = 0; k < D; ++k)
                    if (t.a_req[(size_t)k * t.lda + ask] > std::max<int64_t>(dirty_ub[k], 0)) { may_fit = false; break; }
            if (may_fit) {
                int64_t seen[CMAX_D];
                for (int k = 0; k < D; ++k) seen[k] = INT64_MIN;
                RowSkip& rs = rskip[(size_t)ri];
                if (skip_active && rs.skip.w != 0) {
                    if (ins_log.size() - rs.seen > 64) rs.skip = DirtyRef();   // too much to replay: walk from the front again
                    else
                        for (size_t j = rs.seen; j < ins_log.size(); ++j) {
                            const uint32_t n = ins_log[j];
                            NodeView v = node(n);
                            if (!v.dirty() || v.retired()) continue;
                            const DirtyRef now(v.key(), v.rank(), n);
                            if (now < rs.skip && fits_now(n, ask)) rs.skip = now;
                        }
                }
                rs.seen = (uint32_t)ins_log.size();
                const bool from_start = rs.skip.w == 0;
                const DirtyRef* d = from_start ? dirty.first(cur) : dirty.seek(cur, rs.skip);
                uint32_t misses = 0;
                for (; d && *d < bound; d = dirty.next(cur)) {
                    ++dbg[1];
                    // re-evaluated from the (cache-resident) working copy rather than from the bitmap row, whose lines
                    // were just DMA-written and are cold
                    if (fits_now(d->node(), ask)) { chosen = d->node(); at_cursor = true; break; }
                    ++misses;
                    const int64_t* hh = hot.data() + (size_t)d->node() * hs + 4;   // cap
                    for (int k = 0; k < D; ++k) seen[k] = std::max(seen[k], hh[k]);
                }
                if (d == nullptr && from_start) for (int k = 0; k < D; ++k) dirty_ub[k] = seen[k];   // saw every touched node: exact
                if (misses >= 8 || !from_start) {
                    // everything from the old frontier up to where the walk stopped does not fit this signature
                    rs.skip = (d && *d < bound) ? *d : bound;
                    skip_active = true;
                }
            }
            const unsigned long long tc2 = profile ? commit_tsc() : 0;
            if (chosen != CNONE) ++dbg[2];
            if (chosen == CNONE && posA != CNONE) chosen = bound.node();
            consumed = (size_t)i + 1;
            if (chosen == CNONE) {
                if (in_gang) {
                    // roll the gang back: undo its commits newest-first, void its results, skip its remaining members
                    for (auto it = undo.rbegin(); it != undo.rend(); ++it) {
                        const uint32_t n = it->node;
                        NodeView un = node(n);
                        if (un.retired()) {   // it was taken out of the index when this gang filled it: it is near the back
                            const DirtyRef r(un.key(), un.rank(), n);
                            for (size_t x = retired_refs.size(); x-- > 0;)
                                if (retired_refs[x] == r) { retired_refs.erase(retired_refs.begin() + (long)x); break; }
                            un.set_retired(false);
                        } else {
                            dirty.erase(DirtyRef(un.key(), un.rank(), n));
                        }
                        for (int k = 0; k < D; ++k) un.avail()[k] = it->old_avail[k];
                        un.recap();
                        un.key() = it->old_key;
                        if (it->was_dirty) {
                            dirty.insert(DirtyRef(it->old_key, un.rank(), n));
                            if (skip_active) ins_log.push_back(n);   // its availability went back up: frontiers must re-check it
                            for (int k = 0; k < D; ++k) dirty_ub[k] = std::max(dirty_ub[k], un.cap()[k]);   // it came back
                        } else {
                            un.set_dirty(false);
                            dirty_list.pop_back();
                            const uint32_t pos = it->pos;
                            dirty_words[pos >> 5] &= ~(1u << (pos & 31));
                            front = std::min(front, (int)(pos >> 5));
                        }
                    }
                    undo.clear();
                    int g1 = i + 1;
                    while (g1 < B && same_gang(ask, batch[(size_t)g1])) ++g1;
                    for (int x = gang_begin; x < g1; ++x) result[(size_t)x] = CNONE;
                    consumed = (size_t)g1;
                    i = g1 - 1;
                }
                if (!insensitive) stop = true;
                continue;
            }
            result[(size_t)i] = chosen;
            // commit: available -= request, re-score, move inside the touched order
            NodeView cv = node(chosen);
            int64_t* h = cv.avail();
            if (in_gang) {
                Undo u; u.node = chosen; u.pos = posA; u.old_key = cv.key(); u.was_dirty = cv.dirty();
                for (int k = 0; k < D; ++k) u.old_avail[k] = h[k];
                undo.push_back(u);
            }
            if (cv.dirty()) {
                if (at_cursor) dirty.erase_at(cur);
                else dirty.erase(DirtyRef(cv.key(), cv.rank(), chosen));
                ++dbg[3];
            }
            const unsigned long long tc3 = profile ? commit_tsc() : 0;
            for (int k = 0; k < D; ++k) h[k] -= t.a_req[(size_t)k * t.lda + ask];
            cv.recap();
            const double sc = yk_node_score(D, t.policy, t.w, cv.total(), h, 1);
            const uint64_t nk = yk_key_bits(sc);
            if (nk == YK_KEY_NAN) return -5;
            const unsigned long long tc4 = profile ? commit_tsc() : 0;
            cv.key() = nk;
            bool spent = false;   // below the cycle's smallest request somewhere: no pending ask can ever use it again
            for (int k = 0; k < D; ++k) spent = spent || cv.cap()[k] < cycle_min_req[k];
            if (spent) {
                retired_refs.push_back(DirtyRef(nk, cv.rank(), chosen));
            } else {
                dirty.insert(DirtyRef(nk, cv.rank(), chosen));
                if (skip_active) ins_log.push_back(chosen);
            }
            if (!cv.dirty()) {
                if (!spent) for (int k = 0; k < D; ++k) dirty_ub[k] = std::max(dirty_ub[k], cv.cap()[k]);
                cv.set_dirty(true);
                dirty_list.push_back(chosen);
                const uint32_t pos = posA;   // an untouched node can only have come from the clean scan (A)
                dirty_words[pos >> 5] |= 1u << (pos & 31);
            }
            if (spent) cv.set_retired(true);
            if (profile) {
                const unsigned long long tc5 = commit_tsc();
                prof[0] += tc1 - tc0; prof[1] += tc2 - tc1; prof[2] += tc3 - tc2; prof[3] += tc4 - tc3; prof[4] += tc5 - tc4; prof[5] += 1;
            }
        }
        return 0;
    }

    // Epoch end: new node order = merge(previous order minus the touched positions, touched nodes by their new keys).
    // Both inputs are sorted arrays of (key, rank, node) words, so this is one streaming merge; out_nodes receives the
    // node of every new position (what the device's gather needs).  Returns the number of touched nodes.
    int merge_order(uint32_t* out_nodes, int nlive) {
        const int nd = (int)dirty_list.size();
        std::vector<DirtyRef>& ds = dirty_sorted;
        ds.clear();
        dirty.for_each([&](const DirtyRef& r) { ds.push_back(r); });
        if (!retired_refs.empty()) {   // the retired nodes come back into the order under their final keys
            std::sort(retired_refs.begin(), retired_refs.end());
            const size_t mid = ds.size();
            ds.insert(ds.end(), retired_refs.begin(), retired_refs.end());
            std::inplace_merge(ds.begin(), ds.begin() + (long)mid, ds.end());
        }
        const DirtyRef* in = oref[ocur].data();
        DirtyRef* out = oref[ocur ^ 1].data();
        const size_t nds = ds.size();
        size_t j = 0;
        int o = 0, p = 0, removed = 0;   // removed = touched positions passed over in the old order so far
        while (p < nlive) {
            if ((dirty_words[(size_t)p >> 5] >> (p & 31)) & 1u) { ++p; ++removed; continue; }
            if (j >= nds && removed == nd) {
                // every touched node has been taken out and put back: the rest of the order is unchanged
                memcpy(out + o, in + p, sizeof(DirtyRef) * (size_t)(nlive - p));
                for (int x = p; x < nlive; ++x) out_nodes[o + (x - p)] = in[x].node();
                o += nlive - p;
                p = nlive;
                break;
            }
            const DirtyRef c = in[p];
            while (j < nds && ds[j] < c) { out[o] = ds[j]; out_nodes[o++] = ds[j].node(); ++j; }
            out[o] = c; out_nodes[o++] = c.node();
            ++p;
        }
        while (j < nds) { out[o] = ds[j]; out_nodes[o++] = ds[j].node(); ++j; }
        ocur ^= 1;
        return nd;
    }
};

}  // namespace yk
