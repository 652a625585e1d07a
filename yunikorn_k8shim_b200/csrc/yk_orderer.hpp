// yk_orderer.hpp -- host-side ordering engine: which pending ask does the next schedule() pass try?
//
// Restates, incrementally, what yunikorn-core re-derives from scratch on every pass [EXT, SURVEY A.1/a14]:
//   Queue.TryAllocate: parent -> sortQueues() (fair: DRF share of allocated/guaranteed ascending, then larger
//   pending, children without pending filtered out); leaf -> getHeadRoom() then sortApplications()
//   (fifo: max pending ask priority desc, submission time asc) -> Application.tryAllocate: sortedRequests
//   (priority desc, create time asc), skip asks that exceed the queue headroom.
// The node walk itself (tryNodes) is the device's job.  Because the order of passes does not depend on WHICH
// node an ask lands on, only on WHETHER it was placed, the orderer runs ahead speculatively: fill() returns
// the asks of the next passes assuming each one is placed; if the device reports that ask j found no node,
// rewind() restores the state before the batch and replays the first j decisions.  When the order cannot
// depend on placement at all (one leaf with pending asks, no quota on its chain, fifo, one priority level)
// the batch is "placement-insensitive" and failures do not cut it short.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <map>
#include <set>
#include <tuple>
#include <vector>

namespace yk {

constexpr uint32_t NONE = 0xFFFFFFFFu;
constexpr int64_t UNSET = -1;
enum : uint8_t { ST_PENDING = 0, ST_ALLOCATED = 1, ST_NOFIT = 2, ST_SKIPPED = 3, ST_SLOWPATH = 4, ST_INVALID = 5,
                 ST_TENTATIVE = 100, ST_ABSENT = 255 };

struct Tables {   // views into the engine's host tables
    int D = 0;
    uint32_t maxA = 0, maxP = 0, nq = 0;
    const int64_t* a_req = nullptr;      // [D][maxA]
    const int32_t* a_prio = nullptr;
    const int64_t* a_create = nullptr;
    const uint32_t* a_app = nullptr;
    const uint32_t* a_flags = nullptr;
    const uint8_t* a_cause = nullptr;    // optional: per ask 0, ST_SLOWPATH (flag bit 0) or ST_INVALID (request not strictly > 0), kept by the
                                         // owner of the tables where asks are upserted; null = derived from a_flags / a_req on the fly
    const uint32_t* a_gang = nullptr;    // NONE or gang id (all-or-nothing group inside one application)
    uint8_t* a_state = nullptr;          // ST_*
    const uint32_t* p_queue = nullptr;
    const int64_t* p_submit = nullptr;
    const uint8_t* p_present = nullptr;
    const uint32_t* q_parent = nullptr;
    const int64_t* q_guar = nullptr;     // [D][nq]
    const int64_t* q_max = nullptr;      // [D][nq]
    int64_t* q_alloc = nullptr;          // [D][nq] persistent allocated (updated at finish())
    int64_t* p_alloc = nullptr;          // [D][maxP] persistent per-application allocated (may be null)
    const uint8_t* q_sort = nullptr;
    const int32_t* q_prio_offset = nullptr;   // [nq] queue property priority.offset; null = all 0
    const uint8_t* q_prio_fence = nullptr;    // [nq] 1 = priority.policy fence: the parent sees only the offset; null = none
    // user / group resource limits (the core's queue `limits:` [EXT ugm]; the shim sends the user with every application,
    // pkg/cache/application.go:430): entry l = user ul_user[l] may hold at most ul_max[.][l] below queue ul_queue[l]
    const uint32_t* p_user = nullptr;         // [maxP] user index or NONE; null = no users
    uint32_t n_ul = 0;
    const uint32_t* ul_queue = nullptr;       // [n_ul]
    const uint32_t* ul_user = nullptr;        // [n_ul]
    const int64_t* ul_max = nullptr;          // [D][n_ul], UNSET = not limited
    int64_t* ul_alloc = nullptr;              // [D][n_ul] persistent: what the user holds there (updated at finish())
};

inline bool strictly_gt_zero(const int64_t* v, int d) {
    bool pos = false;
    for (int k = 0; k < d; ++k) { if (v[k] < 0) return false; if (v[k] > 0) pos = true; }
    return pos;
}

// What keeps ask a out of the passes whatever the cluster looks like (Tables::a_cause): the slow-path flag, or a request
// (column-major, leading dimension lda) that is not strictly greater than zero ([EXT] preAllocateCheck)
inline uint8_t ask_cause(int D, const int64_t* a_req, size_t lda, const uint32_t* a_flags, uint32_t a) {
    if (a_flags[a] & 1u) return ST_SLOWPATH;
    int64_t rq[8];
    for (int k = 0; k < D; ++k) rq[k] = a_req[(size_t)k * lda + a];
    return strictly_gt_zero(rq, D) ? 0 : ST_INVALID;
}

class Orderer {
public:
    struct QState {
        int64_t alloc[8], pending[8];
        int64_t npend = 0, live = 0;
        double shares[8];
        bool shares_ok = false;
        int32_t prio = INT32_MIN;   // Queue.GetCurrentPriority: highest priority among the asks still pending below it
        bool prio_ok = false;
    };
    struct AState {
        uint32_t head = 0;       // first ask not allocated/tentative
        int64_t npend = 0, live = 0;
        int32_t key_prio = 0;
        bool in_set = false;
        int64_t alloc[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // allocated to the application (fair leaf ordering)
    };
    // application order inside a leaf: (-max pending priority, [fair leaves: allocation shares against the
    // queue's guaranteed resource, largest first], submission time, app index).  fifo leaves keep sh all zero.
    struct AppKey {
        int64_t negprio; double sh[8]; int64_t submit; uint32_t app;   // 64-bit: -INT32_MIN must not wrap
        bool operator<(const AppKey& o) const {
            if (negprio != o.negprio) return negprio < o.negprio;
            for (int k = 0; k < 8; ++k) if (sh[k] != o.sh[k]) return sh[k] < o.sh[k];
            if (submit != o.submit) return submit < o.submit;
            return app < o.app;
        }
    };
    AppKey make_key(uint32_t p) const {
        AppKey k;
        k.negprio = -(int64_t)ap[p].key_prio; k.submit = t.p_submit[p]; k.app = p;
        for (int i = 0; i < 8; ++i) k.sh[i] = 0.0;
        const uint32_t leaf = t.p_queue[p];
        if (t.q_sort[leaf] == 1) {   // fair
            double tmp[8];
            for (int i = 0; i < t.D; ++i) {
                const int64_t v = ap[p].alloc[i], g = t.q_guar[(size_t)i * t.nq + leaf];
                tmp[i] = (v == 0) ? 0.0 : (g <= 0 ? (double)v : (double)v / (double)g);
            }
            std::sort(tmp, tmp + t.D);
            for (int i = 0; i < t.D; ++i) k.sh[i] = tmp[t.D - 1 - i];   // largest first
        }
        return k;
    }

    Tables t;
    std::vector<QState> q;
    std::vector<std::vector<uint32_t>> q_children, q_apps;
    std::vector<std::set<AppKey>> q_set;
    std::vector<std::vector<uint32_t>> q_sorted, q_changed;   // per parent: cached child order, children to re-position
    std::vector<uint8_t> q_sorted_ok;
    std::vector<uint8_t> q_has_quota;                          // some queue on the chain root..q has a max set
    // queue priorities (parents sort their children by priority first, then by share: sortQueuesByPriorityAndFairness
    // [EXT]).  uniform_prio: every pending ask of the cycle has the same priority, so none of this can matter and it is
    // skipped.  Otherwise every leaf keeps {priority of an application's best pending ask -> how many such applications}.
    bool uniform_prio = true;
    std::vector<std::map<int32_t, int>> q_prio_cnt;
    std::vector<int64_t> ua;                        // [n_ul][8] held under each user-limit entry, this cycle
    std::vector<std::vector<uint32_t>> ap_ul;       // application -> the entries that apply to it
    bool any_ul = false;                            // some application of the cycle has a user limit on its chain
    std::vector<AState> ap;
    std::vector<std::vector<uint32_t>> ap_asks;
    std::vector<uint32_t> a_pos;      // ask -> index in its app list
    bool insensitive = false;
    std::vector<uint32_t> static_order; size_t static_next = 0;
    std::vector<uint32_t> static_apps, sa_mem; size_t sa_app = 0, sa_pos = 0;   // where extend_static() stands
    bool oversize_gang = false;   // a gang larger than the batch capacity was met: the caller must raise its batch size
    uint64_t slow_seen = 0;
    std::vector<uint32_t> slow_list;

    // ---- snapshot for rewind: one per in-flight batch ----
    struct Snap {
        std::vector<QState> q;
        std::vector<AState> ap;
        std::vector<std::set<AppKey>> sets;
        std::vector<std::map<int32_t, int>> prio_cnt;
        std::vector<int64_t> ua;
        std::vector<std::pair<uint32_t, uint8_t>> journal;   // (ask, previous state) written while the batch was filled
        size_t slow_mark = 0;
        bool valid = false;
    };
    std::vector<std::pair<uint32_t, uint8_t>>* jr = nullptr;   // where set_state logs (the batch being filled)

    int D() const { return t.D; }
    int64_t req(uint32_t a, int k) const { return t.a_req[(size_t)k * t.maxA + a]; }

    void begin_cycle(const std::vector<uint32_t>& pending_asks) {
        const int d = t.D;
        q.assign(t.nq, QState());
        q_children.assign(t.nq, {});
        q_apps.assign(t.nq, {});
        q_set.assign(t.nq, {});
        q_sorted.assign(t.nq, {}); q_changed.assign(t.nq, {}); q_sorted_ok.assign(t.nq, 0);
        q_has_quota.assign(t.nq, 0);
        q_prio_cnt.assign(t.nq, {});
        for (uint32_t i = 0; i < t.nq; ++i) {
            for (int k = 0; k < d; ++k) { q[i].alloc[k] = t.q_alloc[(size_t)k * t.nq + i]; q[i].pending[k] = 0; }
            if (i > 0) q_children[t.q_parent[i]].push_back(i);
            bool own = false;
            for (int k = 0; k < d; ++k) if (t.q_max[(size_t)k * t.nq + i] != UNSET) own = true;
            q_has_quota[i] = own || (i > 0 && q_has_quota[t.q_parent[i]]);   // parent[i] < i: already computed
        }
        ap.assign(t.maxP, AState());
        if (ap_asks.size() < t.maxP) ap_asks.resize(t.maxP);
        for (auto& v : ap_asks) v.clear();
        a_pos.assign(t.maxA, 0);
        slow_list.clear();
        for (uint32_t a : pending_asks) ap_asks[t.a_app[a]].push_back(a);
        int32_t prio0 = 0; bool have_prio = false, one_prio = true;
        for (uint32_t p = 0; p < t.maxP; ++p) {
            auto& v = ap_asks[p];
            if (v.empty()) continue;
            auto less = [&](uint32_t l, uint32_t r) {
                if (t.a_prio[l] != t.a_prio[r]) return t.a_prio[l] > t.a_prio[r];
                if (t.a_create[l] != t.a_create[r]) return t.a_create[l] < t.a_create[r];
                return l < r;
            };
            if (!std::is_sorted(v.begin(), v.end(), less)) std::sort(v.begin(), v.end(), less);
            AState& A = ap[p];
            int64_t nlive = 0;
            for (uint32_t i = 0; i < v.size(); ++i) {
                uint32_t a = v[i];
                a_pos[a] = i;
                if (!have_prio) { prio0 = t.a_prio[a]; have_prio = true; }
                else if (t.a_prio[a] != prio0) one_prio = false;
                if (t.a_state[a] == ST_PENDING) ++nlive;
            }
            A.npend = (int64_t)v.size();
            A.live = nlive;
            for (uint32_t qq = t.p_queue[p]; qq != NONE; qq = t.q_parent[qq]) {   // once per application, not per ask
                q[qq].npend += (int64_t)v.size();
                q[qq].live += nlive;
            }   // (the queues' pending RESOURCES are summed below, and only when the order can depend on them)
            q_apps[t.p_queue[p]].push_back(p);
            A.key_prio = t.a_prio[v[0]];
            ++q_prio_cnt[t.p_queue[p]][A.key_prio];
            if (t.p_alloc) for (int k = 0; k < d; ++k) A.alloc[k] = t.p_alloc[(size_t)k * t.maxP + p];
            if (A.live > 0) { q_set[t.p_queue[p]].insert(make_key(p)); A.in_set = true; }
        }
        // user limits: which entries apply to which application (its user, a queue on its chain)
        ua.assign((size_t)t.n_ul * 8, 0);
        if (ap_ul.size() < t.maxP) ap_ul.resize(t.maxP);
        bool any_limit = false;
        if (t.n_ul || any_ul) for (uint32_t p = 0; p < t.maxP; ++p) {
            ap_ul[p].clear();
            if (!t.n_ul || !t.p_user || ap_asks[p].empty() || t.p_user[p] == NONE) continue;
            for (uint32_t l = 0; l < t.n_ul; ++l) {
                if (t.ul_user[l] != t.p_user[p]) continue;
                for (uint32_t qq = t.p_queue[p]; qq != NONE; qq = t.q_parent[qq])
                    if (qq == t.ul_queue[l]) { ap_ul[p].push_back(l); any_limit = true; break; }
            }
        }
        for (uint32_t l = 0; l < t.n_ul; ++l) for (int k = 0; k < d; ++k) ua[(size_t)l * 8 + k] = t.ul_alloc ? t.ul_alloc[(size_t)k * t.n_ul + l] : 0;
        any_ul = any_limit;
        // placement-insensitive?  one leaf with pending asks, fifo, no max on its chain, one priority level
        int leaves = 0; uint32_t leaf = NONE;
        for (uint32_t i = 0; i < t.nq; ++i)
            if (q_children[i].empty() && q[i].npend > 0) { ++leaves; leaf = i; }
        uniform_prio = one_prio;   // ... and no queue shifts or fences priorities
        for (uint32_t i = 0; i < t.nq && uniform_prio; ++i)
            if ((t.q_prio_offset && t.q_prio_offset[i] != 0) || (t.q_prio_fence && t.q_prio_fence[i])) uniform_prio = false;
        insensitive = false;
        if (leaves == 1 && one_prio && t.q_sort[leaf] == 0) {
            bool quota = false;
            for (uint32_t qq = leaf; qq != NONE; qq = t.q_parent[qq])
                for (int k = 0; k < d; ++k) if (t.q_max[(size_t)k * t.nq + qq] != UNSET) quota = true;
            insensitive = !quota && !any_limit;   // a user limit makes headroom depend on what was placed, like a quota
        }
        if (!insensitive)   // pending resources per queue (fair-share ties, headroom bookkeeping): a placement-insensitive order never reads them
            for (uint32_t p = 0; p < t.maxP; ++p) {
                const auto& v = ap_asks[p];
                if (v.empty()) continue;
                int64_t psum[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                for (uint32_t a : v) for (int k = 0; k < d; ++k) psum[k] += req(a, k);
                for (uint32_t qq = t.p_queue[p]; qq != NONE; qq = t.q_parent[qq])
                    for (int k = 0; k < d; ++k) q[qq].pending[k] += psum[k];
            }
        static_order.clear();
        static_next = 0;
        static_apps.clear();
        sa_app = sa_pos = 0;
        if (insensitive)   // the whole cycle's pass order is known up front: apps in set order, asks in app order;
            for (const AppKey& k : q_set[leaf]) static_apps.push_back(k.app);   // it is materialised batch by batch (extend_static)
    }

    // placement-insensitive cycles: append to static_order until `want` entries are waiting (or nothing is left).
    // Same walk the reference's passes would do: applications in leaf order, asks in application order; an ask that can
    // never be tried gets its cause; a gang's pending members follow its first member (marked TENTATIVE so the walk does
    // not meet them again; confirm / fail_in_place / finish give them their final state), one bad member sinks the gang.
    void extend_static(size_t want) {
        const int d = t.D;
        auto cause_of = [&](uint32_t a) -> uint8_t { return t.a_cause ? t.a_cause[a] : ask_cause(d, t.a_req, t.maxA, t.a_flags, a); };
        static_order.reserve(std::min<size_t>(static_order.size() + (want == (size_t)-1 ? (size_t)t.maxA : want), (size_t)t.maxA + 1));
        while (static_order.size() - static_next < want && sa_app < static_apps.size()) {
            const auto& v = ap_asks[static_apps[sa_app]];
            if (sa_pos >= v.size()) { ++sa_app; sa_pos = 0; continue; }
            const uint32_t a = v[sa_pos++];
            if (t.a_state[a] != ST_PENDING) continue;
            if (t.a_gang[a] == NONE) {
                const uint8_t c = cause_of(a);
                if (c) { if (c == ST_SLOWPATH) slow_list.push_back(a); t.a_state[a] = c; continue; }
                static_order.push_back(a);
                continue;
            }
            // a gang member: the first cause among the members (in ask order) sinks every member, all or nothing
            sa_mem.clear();
            uint8_t gc = 0;
            for (uint32_t m : v)
                if (t.a_gang[m] == t.a_gang[a] && t.a_state[m] == ST_PENDING) { sa_mem.push_back(m); if (!gc) gc = cause_of(m); }
            for (uint32_t m : sa_mem) {
                if (gc) { if (gc == ST_SLOWPATH && (t.a_flags[m] & 1u)) slow_list.push_back(m); t.a_state[m] = gc; }
                else { t.a_state[m] = ST_TENTATIVE; static_order.push_back(m); }
            }
        }
    }

    // Next asks in pass order, assuming every one is placed: at most cap_batch of them, and never past
    // cap_user bindings (max_bindings).  A gang is never split: it goes whole into this batch or the next.
    size_t fill(size_t cap_batch, size_t cap_user, std::vector<uint32_t>& batch, Snap& snap) {
        oversize_gang = false;
        batch.clear();
        snap.valid = false;
        if (insensitive) {
            extend_static(cap_batch == (size_t)-1 ? cap_batch : cap_batch + 1);   // one more than fits: the loop below ends on capacity
            while (static_next < static_order.size()) {
                const uint32_t a = static_order[static_next];
                if (t.a_gang[a] == NONE) {   // a stretch of plain asks: one copy
                    const size_t room = std::min(cap_user, cap_batch) - std::min(std::min(cap_user, cap_batch), batch.size());
                    size_t len1 = 0;
                    const size_t lim = std::min(room, static_order.size() - static_next);
                    while (len1 < lim && t.a_gang[static_order[static_next + len1]] == NONE) ++len1;
                    if (len1 == 0) {   // capacity reached: same outcome as the one-entry case below
                        if (batch.size() + 1 > cap_user) break;
                        if (batch.empty()) oversize_gang = true;
                        break;
                    }
                    batch.insert(batch.end(), static_order.begin() + static_next, static_order.begin() + static_next + len1);
                    static_next += len1;
                    continue;
                }
                size_t len = 1;
                if (t.a_gang[a] != NONE)
                    while (static_next + len < static_order.size() && t.a_gang[static_order[static_next + len]] == t.a_gang[a] &&
                           t.a_app[static_order[static_next + len]] == t.a_app[a]) ++len;
                if (batch.size() + len > cap_user) break;                       // max_bindings reached
                if (batch.size() + len > cap_batch) { if (batch.empty()) oversize_gang = true; break; }
                batch.insert(batch.end(), static_order.begin() + static_next, static_order.begin() + static_next + len);
                static_next += len;
            }
            return batch.size();
        }
        snap.journal.clear(); snap.slow_mark = slow_list.size();
        snap.q = q; snap.ap = ap; snap.sets = q_set; snap.ua = ua; snap.valid = true;   // only placement-sensitive orders ever rewind
        if (!uniform_prio) snap.prio_cnt = q_prio_cnt;
        jr = &snap.journal;
        while (step(cap_batch, cap_user, batch)) {}
        jr = nullptr;
        return batch.size();
    }

    // The device placed batch[0..j) and found no node for the ask (or gang) starting at batch[j]: restore the
    // state before the batch, replay the first j decisions, mark the failed ask / gang.
    // `later` = the snapshot of a batch filled after this one (speculatively, already in flight) or null: it is undone too.
    void rewind(Snap& snap, Snap* later, const std::vector<uint32_t>& batch, size_t j) {
        if (later && later->valid) {
            for (auto it = later->journal.rbegin(); it != later->journal.rend(); ++it) t.a_state[it->first] = it->second;
            later->journal.clear();
            later->valid = false;
        }
        for (auto it = snap.journal.rbegin(); it != snap.journal.rend(); ++it) t.a_state[it->first] = it->second;
        snap.journal.clear();
        q = snap.q; ap = snap.ap; q_set = snap.sets; ua = snap.ua; slow_list.resize(snap.slow_mark);
        if (!uniform_prio) q_prio_cnt = snap.prio_cnt;
        snap.valid = false;
        jr = nullptr;
        std::fill(q_sorted_ok.begin(), q_sorted_ok.end(), 0);
        for (auto& v : q_changed) v.clear();
        std::vector<uint32_t> replay;
        while (replay.size() < j && step(j, (size_t)-1, replay)) {}
        // passes that add nothing (a gang sunk by its queue-side checks) may sit between entry j-1 and entry j
        uint32_t a = select(0);
        for (int guard = 0; a != NONE && a != batch[j] && guard < (1 << 20); ++guard) {
            const size_t before = replay.size();
            step((size_t)-1, (size_t)-1, replay);
            if (replay.size() != before) break;   // cannot happen: the decisions are deterministic
            a = select(0);
        }
        if (a == NONE) return;
        if (t.a_gang[a] == NONE) { mark_dead(a, ST_NOFIT); return; }
        std::vector<uint32_t> mem;
        gang_members(a, mem);
        for (uint32_t m : mem) mark_dead(m, ST_NOFIT);
    }

    // The batch is given up after its first j entries were decided (all placed, or failed in place): the entries from
    // j on go back to where fill() took them from.  Used when a cycle moves from the device commit to the host commit.
    void unfill(Snap& snap, const std::vector<uint32_t>& batch, size_t j) {
        if (insensitive) { static_next -= batch.size() - j; return; }
        for (auto it = snap.journal.rbegin(); it != snap.journal.rend(); ++it) t.a_state[it->first] = it->second;
        snap.journal.clear();
        q = snap.q; ap = snap.ap; q_set = snap.sets; ua = snap.ua; slow_list.resize(snap.slow_mark);
        if (!uniform_prio) q_prio_cnt = snap.prio_cnt;
        snap.valid = false;
        jr = nullptr;
        std::fill(q_sorted_ok.begin(), q_sorted_ok.end(), 0);
        for (auto& v : q_changed) v.clear();
        std::vector<uint32_t> replay;
        while (replay.size() < j && step(j, (size_t)-1, replay)) {}
    }

    // insensitive batches: ask `a` (tentatively accounted) found no node
    void fail_in_place(uint32_t a) {
        if (insensitive) { t.a_state[a] = ST_NOFIT; return; }
        const int d = t.D;
        uint32_t p = t.a_app[a];
        t.a_state[a] = ST_NOFIT;
        ap[p].npend++;
        for (int k = 0; k < d; ++k) ap[p].alloc[k] -= req(a, k);
        if (any_ul) for (uint32_t l : ap_ul[p]) for (int k = 0; k < d; ++k) ua[(size_t)l * 8 + k] -= req(a, k);
        if (a_pos[a] < ap[p].head) ap[p].head = a_pos[a];
        for (uint32_t qq = t.p_queue[p]; qq != NONE; qq = t.q_parent[qq]) {
            q[qq].npend++;
            for (int k = 0; k < d; ++k) { q[qq].alloc[k] -= req(a, k); q[qq].pending[k] += req(a, k); }
            q[qq].shares_ok = false;
        }
    }

    void confirm(uint32_t a) {
        t.a_state[a] = ST_ALLOCATED;
        if (insensitive)   // static order: accounting is not needed to order, only to persist; the queue chain gets the
            for (int k = 0; k < t.D; ++k) ap[t.a_app[a]].alloc[k] += req(a, k);   // application's total once, in finish()
    }

    void finish() {   // persist queue and application allocations
        if (insensitive)   // gang members queued but never batched (max_bindings cut the cycle) are simply still pending
            for (size_t i = static_next; i < static_order.size(); ++i)
                if (t.a_state[static_order[i]] == ST_TENTATIVE) t.a_state[static_order[i]] = ST_PENDING;
        if (insensitive)
            for (uint32_t p = 0; p < t.maxP; ++p) {
                if (ap_asks[p].empty()) continue;
                int64_t delta[8];
                bool any = false;
                for (int k = 0; k < t.D; ++k) {
                    delta[k] = ap[p].alloc[k] - (t.p_alloc ? t.p_alloc[(size_t)k * t.maxP + p] : 0);
                    any = any || delta[k] != 0;
                }
                if (!any) continue;
                for (uint32_t qq = t.p_queue[p]; qq != NONE; qq = t.q_parent[qq])
                    for (int k = 0; k < t.D; ++k) q[qq].alloc[k] += delta[k];
            }
        if (t.ul_alloc) for (uint32_t l = 0; l < t.n_ul; ++l) for (int k = 0; k < t.D; ++k) t.ul_alloc[(size_t)k * t.n_ul + l] = ua[(size_t)l * 8 + k];
        for (uint32_t i = 0; i < t.nq; ++i)
            for (int k = 0; k < t.D; ++k) t.q_alloc[(size_t)k * t.nq + i] = q[i].alloc[k];
        if (t.p_alloc)
            for (uint32_t p = 0; p < t.maxP; ++p)
                if (!ap_asks[p].empty()) for (int k = 0; k < t.D; ++k) t.p_alloc[(size_t)k * t.maxP + p] = ap[p].alloc[k];
    }

private:
    void gang_members(uint32_t a, std::vector<uint32_t>& mem) {
        mem.clear();
        for (uint32_t m : ap_asks[t.a_app[a]])
            if (t.a_gang[m] == t.a_gang[a] && t.a_state[m] == ST_PENDING) mem.push_back(m);
    }

    // one schedule() pass of the speculation: appends one ask, or one whole gang; false = batch is closed
    bool step(size_t cap_batch, size_t cap_user, std::vector<uint32_t>& batch) {
        if (batch.size() >= cap_batch || batch.size() >= cap_user) return false;
        const uint32_t a = select(0);
        if (a == NONE) return false;
        if (t.a_gang[a] == NONE) { tentative(a); batch.push_back(a); return true; }
        const int d = t.D;
        std::vector<uint32_t> mem;
        gang_members(a, mem);
        // host-side checks of every member, with the headroom shrinking as earlier members are counted.  They come
        // BEFORE the capacity tests (batch size and max_bindings): a gang sunk here needs no room, and the decision must not depend on how the
        // engine happens to cut its batches (rewind replays with a different capacity).
        int64_t hr[8];
        headroom(t.p_queue[t.a_app[a]], hr);
        if (any_ul) user_headroom(t.a_app[a], hr);
        uint8_t cause = 0;
        for (uint32_t m : mem) {
            if (t.a_flags[m] & 1u) { cause = ST_SLOWPATH; break; }
            bool fits = true;
            for (int k = 0; k < d; ++k) if (hr[k] != UNSET && req(m, k) > hr[k]) { fits = false; break; }
            if (!fits) { cause = ST_SKIPPED; break; }
            int64_t rq[8];
            for (int k = 0; k < d; ++k) rq[k] = req(m, k);
            if (!strictly_gt_zero(rq, d)) { cause = ST_INVALID; break; }
            for (int k = 0; k < d; ++k) if (hr[k] != UNSET) hr[k] -= req(m, k);
        }
        if (cause) {
            for (uint32_t m : mem) { if (cause == ST_SLOWPATH && (t.a_flags[m] & 1u)) slow_list.push_back(m); mark_dead(m, cause); }
            return true;   // nothing added, but the pass moved on
        }
        if (batch.size() + mem.size() > cap_user) return false;                 // max_bindings: the cycle ends here
        if (batch.size() + mem.size() > cap_batch) { if (batch.empty()) oversize_gang = true; return false; }
        for (uint32_t m : mem) { tentative(m); batch.push_back(m); }
        return true;
    }

    void set_state(uint32_t a, uint8_t st) {
        if (jr) jr->emplace_back(a, t.a_state[a]);
        t.a_state[a] = st;
    }
    void drop_live(uint32_t a) {
        uint32_t p = t.a_app[a];
        AState& A = ap[p];
        A.live--;
        for (uint32_t qq = t.p_queue[p]; qq != NONE; qq = t.q_parent[qq]) q[qq].live--;
        if (A.live == 0 && A.in_set) {
            q_set[t.p_queue[p]].erase(make_key(p));
            A.in_set = false;
        }
    }
    void mark_dead(uint32_t a, uint8_t st) {
        set_state(a, st);
        drop_live(a);
    }
    void tentative(uint32_t a) {
        const int d = t.D;
        uint32_t p = t.a_app[a];
        AState& A = ap[p];
        set_state(a, ST_TENTATIVE);
        const int32_t prio_before = A.key_prio;   // the application counted under this priority in its leaf (npend > 0)
        A.npend--;
        drop_live(a);   // may take the app out of its leaf's set
        // advance head; re-key the app if its max pending priority or (fair leaf) its allocation changed
        const auto& v = ap_asks[p];
        while (A.head < v.size() && (t.a_state[v[A.head]] == ST_ALLOCATED || t.a_state[v[A.head]] == ST_TENTATIVE)) A.head++;
        if (any_ul) for (uint32_t l : ap_ul[p]) for (int k = 0; k < d; ++k) ua[(size_t)l * 8 + k] += req(a, k);
        const bool fair = t.q_sort[t.p_queue[p]] == 1;
        const int32_t np = A.head < v.size() ? t.a_prio[v[A.head]] : A.key_prio;
        if (np != A.key_prio || fair) {
            auto& S = q_set[t.p_queue[p]];
            if (A.in_set) S.erase(make_key(p));
            A.key_prio = np;
            for (int k = 0; k < d; ++k) A.alloc[k] += req(a, k);
            if (A.in_set) S.insert(make_key(p));
        } else {
            for (int k = 0; k < d; ++k) A.alloc[k] += req(a, k);
        }
        if (!uniform_prio) {   // the leaf's priority census follows the application's best pending ask
            auto& M = q_prio_cnt[t.p_queue[p]];
            auto it = M.find(prio_before);
            if (it != M.end() && --it->second == 0) M.erase(it);
            if (A.npend > 0) ++M[A.key_prio];
        }
        for (uint32_t qq = t.p_queue[p]; qq != NONE; qq = t.q_parent[qq]) {
            QState& Q = q[qq];
            Q.npend--;
            for (int k = 0; k < d; ++k) { Q.alloc[k] += req(a, k); Q.pending[k] -= req(a, k); }
            Q.shares_ok = false;
            Q.prio_ok = false;
            if (t.q_parent[qq] != NONE) q_changed[t.q_parent[qq]].push_back(qq);
        }
    }

    int32_t prio_of(uint32_t i) {
        QState& Q = q[i];
        if (Q.prio_ok) return Q.prio;
        int32_t best = INT32_MIN;
        if (q_children[i].empty()) {
            const auto& M = q_prio_cnt[i];
            if (!M.empty()) best = M.rbegin()->first;
        } else {
            for (uint32_t c : q_children[i]) if (q[c].npend > 0) best = std::max(best, prio_of(c));
        }
        // priorityValueByPolicy [EXT]: the queue's offset, plus what is pending below unless the queue is a fence
        const int64_t off = t.q_prio_offset ? t.q_prio_offset[i] : 0;
        const bool fence = t.q_prio_fence && t.q_prio_fence[i];
        const int64_t v = off + (fence ? 0 : (int64_t)best);
        best = (int32_t)std::min<int64_t>(INT32_MAX, std::max<int64_t>(INT32_MIN, v));
        Q.prio = best;
        Q.prio_ok = true;
        return best;
    }

    void shares_of(uint32_t i) {
        QState& Q = q[i];
        if (Q.shares_ok) return;
        const int d = t.D;
        for (int k = 0; k < d; ++k) {
            int64_t v = Q.alloc[k], g = t.q_guar[(size_t)k * t.nq + i];
            Q.shares[k] = (v == 0) ? 0.0 : (g <= 0 ? (double)v : (double)v / (double)g);
        }
        for (int a = 1; a < d; ++a) {   // d <= 8: insertion sort
            const double v = Q.shares[a];
            int b = a;
            for (; b > 0 && Q.shares[b - 1] > v; --b) Q.shares[b] = Q.shares[b - 1];
            Q.shares[b] = v;
        }
        Q.shares_ok = true;
    }
    int cmp_shares(uint32_t l, uint32_t r) {
        shares_of(l); shares_of(r);
        for (int k = t.D - 1; k >= 0; --k) {
            if (q[l].shares[k] > q[r].shares[k]) return 1;
            if (q[l].shares[k] < q[r].shares[k]) return -1;
        }
        return 0;
    }

    void headroom(uint32_t leaf, int64_t* hr) {
        const int d = t.D;
        if (!q_has_quota[leaf]) { for (int k = 0; k < d; ++k) hr[k] = UNSET; return; }
        uint32_t chain[64]; int n = 0;
        for (uint32_t qq = leaf; qq != NONE && n < 64; qq = t.q_parent[qq]) chain[n++] = qq;
        for (int k = 0; k < d; ++k) hr[k] = UNSET;
        for (int c = n - 1; c >= 0; --c) {
            uint32_t qq = chain[c];
            for (int k = 0; k < d; ++k) {
                int64_t mx = t.q_max[(size_t)k * t.nq + qq];
                if (mx == UNSET) continue;
                int64_t own = mx - q[qq].alloc[k];
                if (own < 0) own = 0;
                hr[k] = (hr[k] == UNSET) ? own : std::min(hr[k], own);
            }
        }
    }

    // the user headroom of the application's user folded into hr [EXT ugm Headroom]: min over the entries that apply
    void user_headroom(uint32_t p, int64_t* hr) {
        const int d = t.D;
        for (uint32_t l : ap_ul[p])
            for (int k = 0; k < d; ++k) {
                const int64_t mx = t.ul_max[(size_t)k * t.n_ul + l];
                if (mx == UNSET) continue;
                int64_t own = mx - ua[(size_t)l * 8 + k];
                if (own < 0) own = 0;
                hr[k] = (hr[k] == UNSET) ? own : std::min(hr[k], own);
            }
    }

    uint32_t select(uint32_t qi) {
        if (q[qi].live <= 0) return NONE;
        const int d = t.D;
        if (q_children[qi].empty()) {
            int64_t hr_queue[8], hr_user[8];
            headroom(qi, hr_queue);
            int64_t* const hr = any_ul ? hr_user : hr_queue;   // without user limits the queue headroom is the headroom
            auto& S = q_set[qi];
            for (auto it = S.begin(); it != S.end();) {
                uint32_t p = it->app;
                ++it;   // advance first: the body may erase the current element
                if (any_ul) { for (int k = 0; k < d; ++k) hr[k] = hr_queue[k]; user_headroom(p, hr); }
                AState& A = ap[p];
                const auto& v = ap_asks[p];
                for (uint32_t i = A.head; i < v.size(); ++i) {
                    uint32_t a = v[i];
                    if (t.a_state[a] != ST_PENDING) continue;
                    if (t.a_gang[a] != NONE) return a;   // a gang member: step() checks the whole gang, all or nothing
                    if (t.a_flags[a] & 1u) { slow_list.push_back(a); mark_dead(a, ST_SLOWPATH); continue; }
                    bool fits = true;
                    for (int k = 0; k < d; ++k) if (hr[k] != UNSET && req(a, k) > hr[k]) { fits = false; break; }
                    if (!fits) { mark_dead(a, ST_SKIPPED); continue; }
                    int64_t rq[8];
                    for (int k = 0; k < d; ++k) rq[k] = req(a, k);
                    if (!strictly_gt_zero(rq, d)) { mark_dead(a, ST_INVALID); continue; }   // preAllocateCheck
                    return a;
                }
            }
            return NONE;
        }
        // parent: children with pending asks in the order a stable insertion sort from index order gives under the
        // fair comparator (= yunikorn-core sortQueues, Go sort.SliceStable for n <= 20).  The sorted list is cached per
        // parent: between two passes only the child on the allocated path changed, so it is taken out and put back;
        // whenever a comparison ties on the shares (where the pending tie-break is only a partial order and the result
        // could depend on the algorithm) the list is rebuilt with the full insertion sort instead.
        std::vector<uint32_t>& srt = q_sorted[qi];
        bool tie = false;
        auto less = [&](uint32_t l, uint32_t r) {
            if (!uniform_prio) {   // priority first, then the shares (sortQueuesByPriorityAndFairness)
                const int32_t pl = prio_of(l), pr = prio_of(r);
                if (pl != pr) return pl > pr;
            }
            const QState& L = q[l];
            const QState& R = q[r];
            const double a = L.shares[d - 1], b = R.shares[d - 1];   // dominant shares decide almost always
            if (a != b) return a < b;
            for (int k = d - 2; k >= 0; --k) if (L.shares[k] != R.shares[k]) return L.shares[k] < R.shares[k];
            tie = true;
            int64_t diff[8];
            for (int k = 0; k < d; ++k) diff[k] = L.pending[k] - R.pending[k];
            if (strictly_gt_zero(diff, d)) return true;
            for (int k = 0; k < d; ++k) diff[k] = -diff[k];
            if (strictly_gt_zero(diff, d)) return false;
            return l < r;
        };
        bool rebuild = !q_sorted_ok[qi];
        for (uint32_t c : q_changed[qi]) shares_of(c);
        if (!rebuild) {
            for (uint32_t c : q_changed[qi]) {   // re-position the children whose key moved since the last pass
                auto it = std::find(srt.begin(), srt.end(), c);
                if (it != srt.end()) srt.erase(it);
                if (q[c].npend <= 0) continue;
                size_t lo = 0, hi = srt.size();   // first position whose element sorts after c (binary search: the
                while (lo < hi) {                 // others are in order; any tie met on the way forces the rebuild)
                    const size_t mid = (lo + hi) / 2;
                    if (less(c, srt[mid])) hi = mid; else lo = mid + 1;
                }
                // equal share vectors sit next to each other: the search may not have compared c with its equals
                auto same = [&](uint32_t x) { return memcmp(q[c].shares, q[x].shares, sizeof(double) * (size_t)d) == 0; };
                if ((lo > 0 && same(srt[lo - 1])) || (lo < srt.size() && same(srt[lo]))) tie = true;
                srt.insert(srt.begin() + lo, c);
            }
            if (tie) rebuild = true;
        }
        if (rebuild) {
            tie = false;
            srt.clear();
            for (uint32_t c : q_children[qi]) if (q[c].npend > 0) { shares_of(c); srt.push_back(c); }
            for (size_t a = 1; a < srt.size(); ++a)
                for (size_t b = a; b > 0 && less(srt[b], srt[b - 1]); --b) std::swap(srt[b], srt[b - 1]);
            // a list built while shares tie stays "not ok" so that it is rebuilt until the tie is gone
            q_sorted_ok[qi] = !tie;
        }
        q_changed[qi].clear();
        const size_t n = srt.size();
        const uint32_t* s = srt.data();
        for (size_t i = 0; i < n; ++i) {
            uint32_t a = select(s[i]);
            if (a != NONE) return a;
        }
        return NONE;
    }
};

}  // namespace yk
