// Host stand-in of the speculative round-commit launch (csrc/yk_spec.h, yk_spec.cuh) next to the engine's own cycle set-up,
// for the CPU test suite.  spec_run builds the device's static order and screen with the shared rules -- std::stable_sort
// stands in for the cub radix sorts, a sequential sum for the cub scan, plain loops for the reductions -- and, on the same
// tables, runs what yk_cycle does on the host: the pending scan, Orderer::begin_cycle, the commit choice
// (yklt::choose_commit under `auto`) and the adoption test of spec_verify.  Test infrastructure.
#include "../../yunikorn_k8shim_b200/csrc/yk_lattice_host.hpp"
#include "../../yunikorn_k8shim_b200/csrc/yk_spec.h"

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

// out_flags: 0 insensitive, 1 choice.device, 2 plan_ready, 3 the plan is one round-eligible stretch over the whole batch,
// 4 adopt (spec_verify: every condition, the element-for-element compare included), 5 scan.maskfree, 6 scan.longest
extern "C" int spec_run(int D, uint32_t nA, uint32_t nP, uint32_t nQ, uint32_t nN, const int64_t* a_req /*[D][nA]*/,
                        const uint64_t* a_tol, const uint64_t* a_need, const uint64_t* a_deny, const uint32_t* a_node,
                        const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app, const uint32_t* a_flags,
                        const uint32_t* a_gang, const uint32_t* a_sigid, const uint8_t* a_state_in, const uint32_t* p_queue,
                        const int64_t* p_submit, const uint8_t* p_present, const uint32_t* q_parent, const int64_t* q_max,
                        const uint8_t* q_sort, const uint64_t* n_taint, uint32_t max_bindings, int rd_min, int un_min,
                        uint32_t* dev_order, uint32_t* dev_words, uint32_t* static_order, uint32_t* n_static,
                        uint32_t* host_batch, uint32_t* n_batch, int64_t* out_flags) {
    std::vector<uint8_t> cause(nA);
    for (uint32_t a = 0; a < nA; ++a) cause[a] = yk::ask_cause(D, a_req, nA, a_flags, a);
    uint64_t taints = 0;
    for (uint32_t n = 0; n < nN; ++n) taints |= n_taint[n];

    // ---- the device: yk_spec_scan_kernel's reductions and keys, the three sorts, the break sums, the screen ----
    uint32_t w[ykspec::W_N] = {0};
    w[ykspec::W_PRIO_MIN] = 0xFFFFFFFFu;
    std::vector<uint64_t> ckey(nA);
    for (uint32_t a = 0; a < nA; ++a) {
        const uint32_t p = a_app[a];
        ckey[a] = ykspec::time_key(a_create[a]);
        if (!ykspec::kept(a_state_in[a], p < nP ? p_present[p] : 0, cause[a])) continue;
        w[ykspec::W_KEPT]++;
        if (!ykspec::plain(a_gang[a], a_need[a], a_deny[a], a_node[a])) w[ykspec::W_BAD] = 1;
        w[ykspec::W_NOTTOL_LO] |= (uint32_t)~a_tol[a]; w[ykspec::W_NOTTOL_HI] |= (uint32_t)(~a_tol[a] >> 32);
        w[ykspec::W_PRIO_MIN] = std::min(w[ykspec::W_PRIO_MIN], ykspec::prio_word(a_prio[a]));
        w[ykspec::W_PRIO_MAX] = std::max(w[ykspec::W_PRIO_MAX], ykspec::prio_word(a_prio[a]));
    }
    w[ykspec::W_TAINT_LO] = (uint32_t)taints; w[ykspec::W_TAINT_HI] = (uint32_t)(taints >> 32);
    std::vector<uint32_t> apps(nP), pos(nP), order(nA);
    for (uint32_t p = 0; p < nP; ++p) apps[p] = p;
    std::stable_sort(apps.begin(), apps.end(), [&](uint32_t x, uint32_t y) { return ykspec::time_key(p_submit[x]) < ykspec::time_key(p_submit[y]); });
    for (uint32_t j = 0; j < nP; ++j) pos[apps[j]] = j;
    for (uint32_t a = 0; a < nA; ++a) order[a] = a;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return ckey[x] < ckey[y]; });
    std::vector<uint32_t> ukey(nA);
    for (uint32_t a = 0; a < nA; ++a) {
        const uint32_t p = a_app[a];
        const bool k = ykspec::kept(a_state_in[a], p < nP ? p_present[p] : 0, cause[a]);
        ukey[a] = ykspec::app_key(k, k ? pos[p] : 0, nP);
    }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return ukey[x] < ukey[y]; });
    const uint32_t n = ykspec::stretch_len(w[ykspec::W_KEPT], max_bindings);
    std::vector<uint32_t> brk(std::max<uint32_t>(n, 1), 0);
    for (uint32_t i = 0; i < n; ++i) brk[i] = (i ? brk[i - 1] : 0) + ykspec::run_break(order.data(), a_sigid, (int)i);
    for (uint32_t i = 0; i < n; ++i) if (ykspec::long_run_at(brk.data(), (int)i, (int)n, un_min)) w[ykspec::W_RUN] = 1;
    ykspec::decide(w, (uint32_t)rd_min, max_bindings);
    for (uint32_t i = 0; i < n; ++i) dev_order[i] = order[i];
    memcpy(dev_words, w, sizeof(w));

    // ---- the host: yk_cycle's pending scan, the orderer's set-up, the commit choice and spec_verify's test ----
    std::vector<uint8_t> state(a_state_in, a_state_in + nA);
    std::vector<int64_t> q_guar((size_t)D * nQ, -1), q_alloc((size_t)D * nQ, 0), p_alloc((size_t)D * nP, 0);
    yk::Orderer o;
    yk::Tables& t = o.t;
    t.D = D; t.maxA = nA; t.maxP = nP; t.nq = nQ;
    t.a_req = a_req; t.a_prio = a_prio; t.a_create = a_create; t.a_app = a_app; t.a_flags = a_flags; t.a_gang = a_gang;
    t.a_cause = cause.data(); t.a_state = state.data(); t.p_queue = p_queue; t.p_submit = p_submit; t.p_present = p_present;
    t.q_parent = q_parent; t.q_guar = q_guar.data(); t.q_max = q_max; t.q_alloc = q_alloc.data(); t.p_alloc = p_alloc.data(); t.q_sort = q_sort;
    yk::CommitTables ct;
    const double weights[8] = {1, 1, 1, 1, 1, 1, 1, 1};
    ct.D = D; ct.policy = 0; ct.w = weights; ct.lda = nA;
    ct.a_req = a_req; ct.a_tol = a_tol; ct.a_need = a_need; ct.a_deny = a_deny; ct.a_node = a_node; ct.a_gang = a_gang; ct.a_app = a_app;
    yklt::Scan scan;
    scan.taints = taints;
    std::vector<uint32_t> pending;
    bool any_gang = false;
    for (uint32_t a = 0; a < nA; ++a) {
        if (state[a] == yk::ST_ABSENT || state[a] == yk::ST_ALLOCATED) continue;
        state[a] = yk::ST_PENDING;
        if (!p_present[a_app[a]]) continue;
        pending.push_back(a);
        any_gang = any_gang || a_gang[a] != yk::NONE;
        scan.add(ct, a_sigid, a);
    }
    std::vector<uint32_t> a_shape(nA, 0);
    scan.done(ct, pending, false, a_shape);
    o.begin_cycle(pending);
    {   // the whole static order, on a copy of the orderer (extend_static rewrites states: a copy of those too)
        std::vector<uint8_t> st2(state);
        yk::Orderer o2 = o;
        o2.t.a_state = st2.data();
        if (o2.insensitive) o2.extend_static((size_t)-1);
        *n_static = (uint32_t)o2.static_order.size();
        std::copy(o2.static_order.begin(), o2.static_order.end(), static_order);
    }
    std::vector<uint32_t> asks, meta(std::max<uint32_t>(nA, 1)), shp(meta.size()), sig(meta.size()), n_rank(std::max<uint32_t>(nN, 1));
    std::vector<int64_t> n_total((size_t)D * std::max<uint32_t>(nN, 1), 1000);
    for (uint32_t k = 0; k < nN; ++k) n_rank[k] = k;
    const std::vector<uint8_t> npresent(std::max<uint32_t>(nN, 1), 1);
    std::vector<ykun::Segment> segs;
    yk::Orderer::Snap snap;
    yk_stats_t st{};
    const bool ranks_unique = true;
    const yklt::ChoiceIn in{o, ct, pending, nN, npresent.data(), n_total.data(), nN, n_rank.data(), &ranks_unique, &any_gang,
                            false, true, false, un_min, rd_min, scan, 64, nA, max_bindings, a_shape.data(), a_sigid, asks, snap,
                            meta.data(), shp.data(), sig.data(), segs, st};
    yklt::Choice choice;
    if (!yklt::choose_commit(in, choice)) return -1;
    const size_t B = asks.size();
    const bool one = segs.size() == 1 && !segs[0].uniform && segs[0].off == 0 && (size_t)segs[0].len == B &&
                     yklt::round_eligible(ct, o.insensitive, taints, asks.data(), B);
    const bool adopt = choice.device && choice.plan_ready && w[ykspec::W_STATUS] == ykspec::GO && w[ykspec::W_COUNT] == B && one &&
                       memcmp(asks.data(), dev_order, 4 * B) == 0;
    std::copy(asks.begin(), asks.end(), host_batch);
    *n_batch = (uint32_t)B;
    out_flags[0] = o.insensitive; out_flags[1] = choice.device; out_flags[2] = choice.plan_ready; out_flags[3] = one;
    out_flags[4] = adopt; out_flags[5] = scan.maskfree; out_flags[6] = (int64_t)scan.longest;
    return 0;
}
