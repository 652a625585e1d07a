// Host emulation of the binpacking fill (csrc/yk_uniform.h, YK_FLAG_BINPACKING_DEVICE) for the CPU test suite: the fill's
// per-item bodies are single-source, so g++ turns the code of un_depth_kernel (L = 1), un_fill_cap_kernel,
// un_fill_decide_kernel, un_fill_select_kernel and un_apply_rekey_kernel into plain loops, with std::stable_sort for the
// cub radix sorts and a sequential sum for the cub scan.  The driver around them is the engine's own: the real ordering
// engine (csrc/yk_orderer.hpp), eligibility with binpacking allowed, and the batch loop, segment loop (every maximal run a
// fill, anything else a hand-off) and uniform-run attempt of csrc/yk_lattice_host.hpp.  Test infrastructure: the product
// only ever runs the kernels.
//
// Where the engine hands the rest of the cycle over to its host commit, this shim runs the same batch loop with a plain
// sequential first fit over the current order (with gang roll-back), as tests/host/lattice_shim.cpp does.
#include "../../yunikorn_k8shim_b200/csrc/yk_lattice_host.hpp"

#include <algorithm>
#include <cstdint>
#include <vector>

static const int32_t* g_q_prio_offset = nullptr;
static const uint8_t* g_q_prio_fence = nullptr;
extern "C" void host_set_queue_priority(const int32_t* offset, const uint8_t* fence) { g_q_prio_offset = offset; g_q_prio_fence = fence; }
// user / group limits for the next run: application users, then the entries [D][n] column-major
static const uint32_t* g_p_user = nullptr; static uint32_t g_n_ul = 0;
static const uint32_t* g_ul_queue = nullptr; static const uint32_t* g_ul_user = nullptr;
static const int64_t* g_ul_max = nullptr; static int64_t* g_ul_alloc = nullptr;
extern "C" void host_set_user_limits(const uint32_t* p_user, uint32_t n, const uint32_t* queue, const uint32_t* user, const int64_t* max, int64_t* alloc) {
    g_p_user = p_user; g_n_ul = n; g_ul_queue = queue; g_ul_user = user; g_ul_max = max; g_ul_alloc = alloc;
}

namespace {

template <int D>
int run_d(uint32_t policy, const double* weights,
          uint32_t nN, const int64_t* n_total, const int64_t* n_avail, const uint64_t* n_taint, const uint64_t* n_label,
          const uint32_t* n_flags, const uint32_t* n_rank,
          uint32_t nA, uint32_t nP, uint32_t nQ, const int64_t* a_req, const uint64_t* a_tol, const uint64_t* a_need,
          const uint64_t* a_deny, const uint32_t* a_node, const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app,
          const uint32_t* a_flags, const uint32_t* a_gang, const uint32_t* p_queue, const int64_t* p_submit,
          const uint32_t* q_parent, const int64_t* q_guar, const int64_t* q_max, int64_t* q_alloc, const uint8_t* q_sort,
          uint32_t batch, uint32_t max_bindings,
          uint32_t* out_ask, uint32_t* out_node, uint32_t* n_out, uint8_t* state_out, int64_t* avail_out, uint64_t* stats_out) {
    if (policy != YK_POLICY_BINPACKING) return 101;
    yk::Orderer o;
    std::vector<uint8_t> state(nA, yk::ST_PENDING), present(nP, 1), npresent(nN, 1);
    std::vector<int64_t> p_alloc((size_t)D * nP, 0);
    o.t.D = D; o.t.maxA = nA; o.t.maxP = nP; o.t.nq = nQ;
    o.t.a_req = a_req; o.t.a_prio = a_prio; o.t.a_create = a_create; o.t.a_app = a_app; o.t.a_flags = a_flags; o.t.a_gang = a_gang;
    std::vector<uint8_t> a_cause(nA, 0);   // the per-ask cause table the engine keeps at upsert time (yk::Tables::a_cause)
    for (uint32_t a = 0; a < nA; ++a) {
        bool pos = false, neg = false;
        for (int k = 0; k < D; ++k) { const int64_t v = a_req[(size_t)k * nA + a]; neg = neg || v < 0; pos = pos || v > 0; }
        a_cause[a] = (a_flags[a] & 1u) ? yk::ST_SLOWPATH : ((neg || !pos) ? yk::ST_INVALID : 0);
    }
    o.t.a_cause = a_cause.data();
    o.t.a_state = state.data(); o.t.p_queue = p_queue; o.t.p_submit = p_submit; o.t.p_present = present.data();
    o.t.q_parent = q_parent; o.t.q_guar = q_guar; o.t.q_max = q_max; o.t.q_alloc = q_alloc; o.t.p_alloc = p_alloc.data(); o.t.q_sort = q_sort;
    o.t.q_prio_offset = g_q_prio_offset; o.t.q_prio_fence = g_q_prio_fence;
    o.t.p_user = g_p_user; o.t.n_ul = g_n_ul; o.t.ul_queue = g_ul_queue; o.t.ul_user = g_ul_user; o.t.ul_max = g_ul_max; o.t.ul_alloc = g_ul_alloc;
    std::vector<uint32_t> pending(nA);
    for (uint32_t i = 0; i < nA; ++i) pending[i] = i;
    o.begin_cycle(pending);
    const bool ins = o.insensitive;

    yk::CommitTables ct;
    ct.D = D; ct.policy = policy; ct.w = weights; ct.lda = nA;
    ct.a_req = a_req; ct.a_tol = a_tol; ct.a_need = a_need; ct.a_deny = a_deny; ct.a_node = a_node; ct.a_gang = a_gang; ct.a_app = a_app;
    const yklt::Eligibility el = yklt::eligible(ct, nN, npresent.data(), n_total, nN, n_rank, pending, nullptr, nullptr, true);
    if (!el.ok) return 100;
    std::vector<uint64_t> a_sig(nA);
    std::vector<uint32_t> a_shape(nA, 0), a_sigid(nA, 0);
    for (uint32_t a = 0; a < nA; ++a) a_sig[a] = yk::ask_signature(ct, a);
    uint32_t n_shapes = 0;
    yklt::assign_shapes(ct, pending, a_shape, &n_shapes);
    yklt::assign_sigs(ct, a_sig.data(), pending, a_sigid);

    // ---- device state: node records and the order (what yk_key_kernel + the radix sort + yk_lt_init_kernel build) ----
    const int RS = (2 * D + 3 + 3) / 4 * 4;
    std::vector<int64_t> rec((size_t)std::max<uint32_t>(nN, 1) * RS, 0);
    std::vector<yklt::Ent> ord0(std::max<uint32_t>(nN, 1));
    for (uint32_t n = 0; n < nN; ++n) {
        int64_t* r = rec.data() + (size_t)n * RS;
        for (int k = 0; k < D; ++k) { r[k] = n_avail[(size_t)k * nN + n]; r[D + k] = n_total[(size_t)k * nN + n]; }
        r[2 * D] = (int64_t)n_taint[n]; r[2 * D + 1] = (int64_t)n_label[n];
        r[2 * D + 2] = (int64_t)(((uint64_t)n_rank[n] << 32) | n_flags[n]);
        ord0[n].key = yk_key_bits(yk_node_score(D, policy, weights, n_total + n, n_avail + n, nN));
        ord0[n].rn = ((uint64_t)n_rank[n] << 32) | n;
        if (ord0[n].key == YK_KEY_NAN) return -5;
    }
    auto ent_lt = [](const yklt::Ent& x, const yklt::Ent& y) { return x.key < y.key || (x.key == y.key && x.rn < y.rn); };
    std::sort(ord0.begin(), ord0.begin() + nN, ent_lt);
    double w[8];
    for (int k = 0; k < 8; ++k) w[k] = k < D ? weights[k] : 0.0;

    // the order must stay exactly: every node once, ascending by (CURRENT key, rank)
    auto order_ok = [&]() -> bool {
        std::vector<uint8_t> seen(nN, 0);
        for (uint32_t p = 0; p < nN; ++p) {
            const uint32_t n = (uint32_t)ord0[p].rn;
            if (n >= nN || seen[n]) return false;
            seen[n] = 1;
            const int64_t* r = rec.data() + (size_t)n * RS;
            if (ord0[p].key != yk_key_bits(yk_node_score(D, policy, weights, r + D, r, 1)) || (ord0[p].rn >> 32) != n_rank[n]) return false;
            if (p > 0 && !ent_lt(ord0[p - 1], ord0[p])) return false;
        }
        return true;
    };
    // plain sequential first fit on the current order (stands in for the engine's host commit after a hand-off)
    auto resort = [&]() {
        for (uint32_t p = 0; p < nN; ++p) {
            const int64_t* r = rec.data() + (size_t)(uint32_t)ord0[p].rn * RS;
            ord0[p].key = yk_key_bits(yk_node_score(D, policy, weights, r + D, r, 1));
        }
        std::sort(ord0.begin(), ord0.begin() + nN, ent_lt);
    };
    auto seq_place = [&](uint32_t ask) -> uint32_t {
        int64_t rq[D];
        for (int k = 0; k < D; ++k) rq[k] = a_req[(size_t)k * nA + ask];
        for (uint32_t p = 0; p < nN; ++p) {
            const uint32_t n = (uint32_t)ord0[p].rn;
            int64_t* r = rec.data() + (size_t)n * RS;
            const uint32_t fl = (uint32_t)(uint64_t)r[2 * D + 2];
            if (!yklt::fits<D>((fl & 1u) && !(fl & 2u), r, r + D, rq)) continue;
            if (!yklt::accepts((uint64_t)r[2 * D], (uint64_t)r[2 * D + 1], n, a_tol[ask], a_need[ask], a_deny[ask], a_node[ask])) continue;
            for (int k = 0; k < D; ++k) r[k] -= rq[k];
            resort();
            return n;
        }
        return yk::CNONE;
    };

    // one fill: the engine's ykun::uniform_run with the kernels of un_fill_d replaced by loops over the same per-item bodies
    std::vector<uint32_t> asks, result, meta(std::max<uint32_t>(nA, 1)), shp(meta.size()), sig(meta.size());
    yk_stats_t st{};
    uint64_t attempts = 0;
    std::vector<uint32_t> byrank(nN);   // the nodes by ascending (NodeID rank, index)
    for (uint32_t i = 0; i < nN; ++i) byrank[i] = i;
    std::sort(byrank.begin(), byrank.end(), [&](uint32_t x, uint32_t y) { return n_rank[x] != n_rank[y] ? n_rank[x] < n_rank[y] : x < y; });
    auto fill = [&](size_t off, size_t R, bool has_gang, int* ust, size_t* consumed) -> int {
        const int nlive = (int)nN;
        const size_t nl = (size_t)nlive;
        std::vector<uint32_t> cnt((size_t)nN, 0), enode(nl), snode(nl), idx(nl);
        std::vector<unsigned long long> ekey(nl), skey(nl), bk(nl), rkey(nl), rrn(nl);
        const uint32_t ask = asks[off];
        ykun::Args a{};
        a.policy = policy;
        for (int k = 0; k < 8; ++k) { a.w[k] = w[k]; a.req[k] = k < D ? a_req[(size_t)k * nA + ask] : 0; }
        a.rec = rec.data(); a.RS = RS; a.nlive = nlive; a.byrank = byrank.data();
        a.tol = a_tol[ask]; a.need = a_need[ask]; a.deny = a_deny[ask]; a.want = a_node[ask];
        a.R = (int)R; a.insensitive = ins ? 1 : 0; a.has_gang = has_gang ? 1 : 0;
        a.ekey = ekey.data(); a.enode = enode.data(); a.skey = skey.data(); a.snode = snode.data();
        a.bk = bk.data(); a.cnt = cnt.data(); a.rkey = rkey.data(); a.rrn = rrn.data();
        a.res = result.data() + off;
        auto attempt = [&](int L, ykun::Globals& g) -> int {
            if (L != 1) return -98;   // a fill generates one key per node
            a.L = 1; a.g = &g;
            g.bkey = ykun::KEY_INF; g.brank = ykun::KEY_INF; g.last_key = 0; g.last_rank = 0; g.valid = 0; g.nan = 0; g.status = ykun::U_RETRY; g.consumed = 0;
            for (int x = 0; x < nlive; ++x) if (ykun::element_item<D>(a, x).nan) g.nan = 1;
            for (size_t x = 0; x < nl; ++x) idx[x] = (uint32_t)x;
            std::stable_sort(idx.begin(), idx.end(), [&](uint32_t x, uint32_t y) { return ekey[x] < ekey[y]; });
            for (size_t x = 0; x < nl; ++x) { skey[x] = ekey[idx[x]]; snode[x] = enode[idx[x]]; }
            unsigned long long sum = 0;
            for (int p = 0; p < nlive; ++p) { ykun::fill_cap_item<D>(a, p); sum += ekey[(size_t)p]; bk[(size_t)p] = sum; }
            ykun::fill_decide(a);
            for (int q = 0; q < (int)R; ++q) ykun::fill_select_item(a, q, g.valid);
            for (int i = 0; i < nlive; ++i) { ykun::apply_item<D>(a, i, g.status); if (ykun::rekey_item<D>(a, i)) g.nan = 2; }
            {   // the order after the fill (what un_reorder builds from the re-keyed entries)
                std::vector<uint32_t> ix(nl);
                for (size_t i = 0; i < nl; ++i) ix[i] = (uint32_t)i;
                std::stable_sort(ix.begin(), ix.end(), [&](uint32_t x, uint32_t y) { return rkey[x] < rkey[y]; });
                for (size_t p = 0; p < nl; ++p) { ord0[p].key = rkey[ix[p]]; ord0[p].rn = rrn[ix[p]]; }
            }
            for (uint32_t c : cnt) if (c) return -99;   // counters must be clean after every fill
            ++attempts;
            return 0;
        };
        const int rc = ykun::uniform_run(D, w, a.req, n_total, nN, byrank.data(), nlive, (int)R, 0, st, attempt, ust, consumed, true);
        if (rc) return rc;
        return *ust == ykun::U_NAN || order_ok() ? 0 : -9;
    };
    std::vector<ykun::Segment> segs;
    auto batch_fn = [&](size_t B, int* status, size_t* consumed) -> int {
        result.assign(B, yk::CNONE);
        return yklt::run_segments(segs, meta.data(), fill, yklt::hand_off, status, consumed);
    };
    // after a hand-off: a plain sequential first fit with gang roll-back, the stand-in for the engine's host commit
    auto sequential = [&](size_t B, int* status, size_t* consumed) -> int {
        result.assign(B, yk::CNONE);
        size_t i = 0;
        bool stop = false;
        while (i < B && !stop) {   // an ask or a whole gang at a time: all of it placed, or none
            size_t g1 = i + 1;
            while (g1 < B && yk::same_gang(o.t, asks[i], asks[g1])) ++g1;
            const std::vector<int64_t> keep(rec);
            size_t x = i;
            while (x < g1 && (result[x] = seq_place(asks[x])) != yk::CNONE) ++x;
            if (x < g1) {
                std::copy(keep.begin(), keep.end(), rec.begin());
                resort();
                std::fill(result.begin() + i, result.begin() + g1, yk::CNONE);
                stop = !ins;
            }
            i = g1;
        }
        *status = stop ? yklt::ST_STOPPED : yklt::ST_DONE;
        *consumed = i;
        return 0;
    };
    uint32_t n = 0;
    auto bind = [&](uint32_t a, uint32_t node) { out_ask[n] = a; out_node[n] = node; ++n; };
    // YK_ERR_RANGE = -5: a NaN score; YK_ERR_ARG = -1: a gang no batch holds; a batch that ended early without a failure
    // is -13 in an insensitive order, -12 in a placement-sensitive one
    auto fail = [&](int code, const char*) { return code == YK_ERR_CUDA ? (ins ? -13 : -12) : code; };

    yk::Orderer::Snap snap;
    bool plan_ready = false, handoff = false;
    yklt::Loop lp{o, ct, a_shape.data(), a_sigid.data(), asks, snap, result, meta.data(), shp.data(), sig.data(), segs, plan_ready,
                  1, nN == 0, batch, max_bindings, n, st};
    size_t bsz = batch;
    if (!yk::fill_batch(o, bsz, batch, max_bindings, asks, snap, st)) return -1;
    int rc = yklt::device_commit(lp, batch_fn, bind, fail, handoff);
    if (!rc && handoff) {   // the engine's path: the rest of the cycle on the host commit, never back on the device
        lp.min_run = 0;
        bsz = batch;
        if (!yk::fill_batch(o, bsz, batch, (size_t)max_bindings - n, asks, snap, st)) return -1;
        rc = yklt::device_commit(lp, sequential, bind, fail, handoff);
    }
    if (rc) return rc;
    o.finish();
    *n_out = n;
    for (uint32_t i = 0; i < nA; ++i) state_out[i] = state[i];
    for (uint32_t nn = 0; nn < nN; ++nn)
        for (int k = 0; k < D; ++k) avail_out[(size_t)k * nN + nn] = rec[(size_t)nn * RS + k];
    if (stats_out) {   // the layout of lattice_shim.cpp's stats_out (the lattice kernel's words stay 0: it never runs here)
        for (int k = 0; k < 6; ++k) stats_out[k] = 0;
        stats_out[6] = st.lattice_handoffs; stats_out[7] = st.batches;
        stats_out[8] = attempts; stats_out[9] = st.uniform_retries; stats_out[10] = st.uniform_asks;
        stats_out[11] = st.uniform_runs; stats_out[12] = st.uniform_elements;
    }
    return 0;
}

}  // namespace

// same argument list as engine_host_run (tests/host/engine_shim.cpp) so that the Python harness is shared; epoch_limit,
// speculate and share_rows do not apply.  Returns 100 when the snapshot is not eligible for the device commit, 101 when its
// node sort is not binpacking.
extern "C" int binpack_host_run(int D, uint32_t policy, const double* weights,
    uint32_t nN, const int64_t* n_total, const int64_t* n_avail, const uint64_t* n_taint, const uint64_t* n_label,
    const uint32_t* n_flags, const uint32_t* n_rank,
    uint32_t nA, uint32_t nP, uint32_t nQ, const int64_t* a_req, const uint64_t* a_tol, const uint64_t* a_need,
    const uint64_t* a_deny, const uint32_t* a_node, const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app,
    const uint32_t* a_flags, const uint32_t* a_gang, const uint32_t* p_queue, const int64_t* p_submit,
    const uint32_t* q_parent, const int64_t* q_guar, const int64_t* q_max, int64_t* q_alloc, const uint8_t* q_sort,
    uint32_t batch, uint32_t /*epoch_limit*/, int /*speculate*/, int /*share_rows*/, uint32_t max_bindings,
    uint32_t* out_ask, uint32_t* out_node, uint32_t* n_out, uint8_t* state_out, int64_t* avail_out, uint64_t* stats_out) {
#define RUN(DD) case DD: return run_d<DD>(policy, weights, nN, n_total, n_avail, n_taint, n_label, n_flags, n_rank, nA, nP, nQ, a_req, a_tol, a_need, a_deny, a_node, a_prio, a_create, a_app, a_flags, a_gang, p_queue, p_submit, q_parent, q_guar, q_max, q_alloc, q_sort, batch, max_bindings, out_ask, out_node, n_out, state_out, avail_out, stats_out);
    switch (D) { RUN(1) RUN(2) RUN(3) RUN(4) RUN(5) RUN(6) RUN(7) RUN(8) default: return -2; }
#undef RUN
}
