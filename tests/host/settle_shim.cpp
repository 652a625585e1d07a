// CPU harness for settling a batch while it is being decided (yklt::settle_ahead / yklt::settle_back,
// csrc/yk_lattice_host.hpp), which the engine does behind the round kernel.  The device commit's batch loop
// (yklt::device_commit) runs one placement-insensitive cycle.  Its batch is decided by a plain sequential first fit over
// the fair node order, and the decided prefix is settled every `chunk` entries, the way the engine settles each prefix the
// round kernel publishes.  With nan_at >= 0 the batch ends on a NaN at that entry after settling what came before it; the
// engine then takes that prefix back, and so does this harness.
// Unlike the device shim, the outputs are written on the NaN error too, so that a test can check what was taken back.
#include "../../yunikorn_k8shim_b200/csrc/yk_lattice_host.hpp"
#include "shim_tables.hpp"

#include <algorithm>
#include <cstdint>
#include <vector>

static int g_chunk = 1, g_nan_at = -1;
extern "C" void settle_set(int chunk, int nan_at) { g_chunk = chunk; g_nan_at = nan_at; }

namespace {

template <int D>
int run_d(uint32_t policy, const double* weights, uint32_t nN, const int64_t* n_total, const int64_t* n_avail, const uint64_t* n_taint,
          const uint64_t* n_label, const uint32_t* n_flags, const uint32_t* n_rank, uint32_t nA, uint32_t nP, uint32_t nQ,
          const int64_t* a_req, const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app, const uint32_t* a_flags,
          const uint32_t* a_gang, const uint32_t* p_queue, const int64_t* p_submit, const uint32_t* q_parent, const int64_t* q_guar,
          const int64_t* q_max, int64_t* q_alloc, const uint8_t* q_sort, uint32_t max_bindings, uint32_t* out_ask,
          uint32_t* out_node, uint32_t* n_out, uint8_t* state_out, int64_t* avail_out, uint64_t* stats_out) {
    yk::Orderer o;
    ShimTables tb;
    wire_orderer(o.t, tb, D, nA, nP, nQ, a_req, a_prio, a_create, a_app, a_flags, a_gang, p_queue, p_submit, q_parent, q_guar, q_max,
                 q_alloc, q_sort);
    std::vector<uint32_t> pending(nA);
    for (uint32_t i = 0; i < nA; ++i) pending[i] = i;
    o.begin_cycle(pending);
    if (!o.insensitive) return -2;
    std::vector<int64_t> app_alloc0((size_t)nP * D);   // the orderer's application totals before anything is settled
    for (uint32_t p = 0; p < nP; ++p) for (int k = 0; k < D; ++k) app_alloc0[(size_t)p * D + k] = o.ap[p].alloc[k];

    // node records, sorted by (current key, NodeID rank) before every placement
    const int RS = yklt::record_words(D);
    std::vector<int64_t> rec((size_t)std::max<uint32_t>(nN, 1) * RS, 0);
    std::vector<yklt::Ent> ord(std::max<uint32_t>(nN, 1));
    {
        std::vector<uint64_t> skey(nN);
        std::vector<uint32_t> snode(nN);
        for (uint32_t n = 0; n < nN; ++n) { skey[n] = 0; snode[n] = n; }
        for (uint32_t p = 0; p < nN; ++p)
            yklt::init_node(D, (int)p, n_total, n_avail, nN, n_taint, n_label, n_flags, n_rank, skey.data(), snode.data(), rec.data(), RS,
                            ord.data());
    }
    auto place = [&](uint32_t ask) -> uint32_t {
        for (uint32_t p = 0; p < nN; ++p) {
            const int64_t* r = rec.data() + (size_t)(uint32_t)ord[p].rn * RS;
            ord[p].key = yk_key_bits(yk_node_score(D, policy, weights, r + D, r, 1));
        }
        std::sort(ord.begin(), ord.begin() + nN, [](const yklt::Ent& x, const yklt::Ent& y) { return yklt::ent_less(x.key, x.rn, y.key, y.rn); });
        int64_t rq[D];
        for (int k = 0; k < D; ++k) rq[k] = a_req[(size_t)k * nA + ask];
        for (uint32_t p = 0; p < nN; ++p) {
            const uint32_t n = (uint32_t)ord[p].rn;
            int64_t* r = rec.data() + (size_t)n * RS;
            const uint32_t fl = (uint32_t)(uint64_t)r[2 * D + 2];
            if (!yklt::fits<D>((fl & 1u) && !(fl & 2u), r, r + D, rq)) continue;
            for (int k = 0; k < D; ++k) r[k] -= rq[k];
            return n;
        }
        return yk::CNONE;
    };

    yk::CommitTables ct;
    ct.D = D; ct.policy = policy; ct.w = weights; ct.lda = nA; ct.a_req = a_req; ct.a_gang = a_gang; ct.a_app = a_app;
    std::vector<uint32_t> asks, result, meta(std::max<uint32_t>(nA, 1)), shp(meta.size()), sig(meta.size()), ids(meta.size(), 0);
    std::vector<ykun::Segment> segs;
    yk::Orderer::Snap snap;
    yk_stats_t st{};
    size_t bsz = nA;
    if (!yk::fill_batch(o, bsz, nA, max_bindings, asks, snap, st)) return -1;
    uint32_t n = 0;
    bool plan_ready = false;
    uint64_t ahead_calls = 0;
    auto bind = [&](uint32_t a, uint32_t node) { out_ask[n] = a; out_node[n] = node; ++n; };
    yklt::Loop lp{o, ct, ids.data(), ids.data(), asks, snap, result, meta.data(), shp.data(), sig.data(), segs, plan_ready, 0, nN == 0,
                  (size_t)nA, max_bindings, n, st};
    auto batch = [&](size_t B, int* status, size_t* consumed) -> int {
        result.assign(B, yk::CNONE);
        *status = yklt::ST_DONE;
        *consumed = B;
        for (size_t i = 0; i < B; ++i) {
            if ((int)i == g_nan_at) { *status = yklt::ST_NAN; *consumed = i; break; }
            result[i] = place(asks[i]);
            if ((i + 1) % (size_t)g_chunk == 0) { yklt::settle_ahead(lp, result.data(), 0, i + 1, bind); ++ahead_calls; }
        }
        if (*status == yklt::ST_NAN) yklt::settle_back(lp, [&](uint32_t) { --n; });
        return 0;
    };
    bool handoff = false;
    const int rc = yklt::device_commit(lp, batch, bind, [&](int code, const char*) { return code; }, handoff);
    if (!rc) o.finish();
    bool app_back = true;   // after a failed batch: the orderer's application totals are what they were
    if (rc) for (uint32_t p = 0; p < nP; ++p) for (int k = 0; k < D; ++k) app_back = app_back && o.ap[p].alloc[k] == app_alloc0[(size_t)p * D + k];
    *n_out = n;
    for (uint32_t i = 0; i < nA; ++i) state_out[i] = tb.state[i];
    for (uint32_t nn = 0; nn < nN; ++nn)
        for (int k = 0; k < D; ++k) avail_out[(size_t)k * nN + nn] = rec[(size_t)nn * RS + k];
    const uint64_t c[] = {st.allocations, st.nofit, ahead_calls, app_back ? 1u : 0u};
    std::copy(c, c + 4, stats_out);
    return rc;
}

}  // namespace

// the argument list of engine_host_run (tests/host/engine_shim.cpp), so that the Python harness is shared; masks, batch,
// epoch_limit, speculate and share_rows do not apply (the whole static order is one batch)
extern "C" int settle_host_run(int D, uint32_t policy, const double* weights,
    uint32_t nN, const int64_t* n_total, const int64_t* n_avail, const uint64_t* n_taint, const uint64_t* n_label,
    const uint32_t* n_flags, const uint32_t* n_rank,
    uint32_t nA, uint32_t nP, uint32_t nQ, const int64_t* a_req, const uint64_t*, const uint64_t*,
    const uint64_t*, const uint32_t*, const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app,
    const uint32_t* a_flags, const uint32_t* a_gang, const uint32_t* p_queue, const int64_t* p_submit,
    const uint32_t* q_parent, const int64_t* q_guar, const int64_t* q_max, int64_t* q_alloc, const uint8_t* q_sort,
    uint32_t, uint32_t, int, int, uint32_t max_bindings,
    uint32_t* out_ask, uint32_t* out_node, uint32_t* n_out, uint8_t* state_out, int64_t* avail_out, uint64_t* stats_out) {
#define RUN(DD) case DD: return run_d<DD>(policy, weights, nN, n_total, n_avail, n_taint, n_label, n_flags, n_rank, nA, nP, nQ, a_req, a_prio, a_create, a_app, a_flags, a_gang, p_queue, p_submit, q_parent, q_guar, q_max, q_alloc, q_sort, max_bindings, out_ask, out_node, n_out, state_out, avail_out, stats_out);
    switch (D) { RUN(1) RUN(2) RUN(3) RUN(4) RUN(5) RUN(6) RUN(7) RUN(8) default: return -2; }
#undef RUN
}
