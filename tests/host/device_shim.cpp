// Host emulation of the device commit for the CPU test suite.  csrc/yk_lattice.h, yk_rounds.h and yk_uniform.h are single
// source -- nvcc turns them into the lattice, round and uniform-run kernels, g++ turns the SAME code into plain loops -- so
// the device commit (lattice sub-runs, rounds, uniform-run attempts, binpacking fills) is checked against the oracle here
// without a GPU.  The driver around them is the engine's own: the ordering engine (csrc/yk_orderer.hpp) and, from
// csrc/yk_lattice_host.hpp, the commit choice, the batch loop, the segment loop, a uniform run's attempts and the per-batch
// routing.
// std::stable_sort stands in for the cub radix sorts and a sequential sum for the cub scan.  After every kernel stand-in the
// shim checks that the node order is exactly "every node once, ascending by (current key, NodeID rank)".
//
// Where the engine hands the rest of the cycle over to its host commit (status HANDOFF), this shim runs the same batch loop
// with a plain sequential first fit over the current order, with gang roll-back.  Test infrastructure: the product only
// ever runs the kernels.
#include "../../yunikorn_k8shim_b200/csrc/yk_lattice_host.hpp"
#include "../../yunikorn_k8shim_b200/csrc/yk_rounds.h"
#include "shim_tables.hpp"

#include <algorithm>
#include <cstdint>
#include <memory>
#include <vector>

// the engine's commit choice: automatic = 1 is `auto` (yklt::choose_commit's cost rule picks the commit and cuts the first
// batch; a cycle it leaves on the host commit returns HOST_COMMIT uncommitted); otherwise the forced `device` choice, with
// batches cut at `batch`, where rounds = 1 routes round-eligible stretches to the round commit as `auto` does and 0 leaves
// every stretch to the lattice kernel; binpacking = 1 is YK_FLAG_BINPACKING_DEVICE
static int g_rounds = 1, g_binpacking = 0, g_auto = 0;
extern "C" void host_set_device(int rounds, int binpacking, int automatic) { g_rounds = rounds; g_binpacking = binpacking; g_auto = automatic; }
// shortest uniform run that takes the uniform-run path (0: never), and how deep the first attempt generates (0: the engine's rule)
static int g_un_min = 0, g_un_depth = 0;
extern "C" void host_set_uniform(int min_run, int first_depth) { g_un_min = min_run; g_un_depth = first_depth; }
// candidates per round (0: ykrd::WCAP), the guard's asks per pass and the fewest pending asks for which a mask-free cycle
// starts on the round commit under `auto` (YK_ROUND_MIN; < 0: the engine's values)
static int g_rd_window = 0, g_rd_guard = -1, g_rd_min = -1;
extern "C" void host_set_rounds(int window, int guard, int min_asks) { g_rd_window = window; g_rd_guard = guard; g_rd_min = min_asks; }

constexpr int INELIGIBLE = 100, HOST_COMMIT = 101;

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
    const bool bp = g_binpacking && policy == YK_POLICY_BINPACKING;
    yk::Orderer o;
    ShimTables tb;
    wire_orderer(o.t, tb, D, nA, nP, nQ, a_req, a_prio, a_create, a_app, a_flags, a_gang, p_queue, p_submit, q_parent, q_guar, q_max,
                 q_alloc, q_sort);
    std::vector<uint32_t> pending(nA);
    for (uint32_t i = 0; i < nA; ++i) pending[i] = i;
    o.begin_cycle(pending);
    const bool ins = o.insensitive;

    yk::CommitTables ct;
    ct.D = D; ct.policy = policy; ct.w = weights; ct.lda = nA;
    ct.a_req = a_req; ct.a_tol = a_tol; ct.a_need = a_need; ct.a_deny = a_deny; ct.a_node = a_node; ct.a_gang = a_gang; ct.a_app = a_app;
    std::vector<uint64_t> a_sig(nA);
    std::vector<uint32_t> a_shape(nA, 0), a_sigid(nA, 0);
    for (uint32_t a = 0; a < nA; ++a) a_sig[a] = yk::ask_signature(ct, a);
    yklt::assign_sigs(ct, a_sig.data(), pending, a_sigid);

    // the engine's commit choice on every node live and every ask pending, in index order; the forced choice fills the first
    // batch at `batch` (the largest batch stands in for the whole static order)
    const bool automatic = g_auto && g_un_min > 0 && (policy == YK_POLICY_FAIR || g_binpacking);
    uint64_t taints = 0;
    for (uint32_t nn = 0; nn < nN; ++nn) taints |= n_taint[nn];
    yklt::Scan scan;
    scan.taints = taints;
    if (automatic) for (uint32_t a : pending) scan.add(ct, a_sigid.data(), a);
    scan.done(ct, pending, !g_auto, a_shape);
    std::vector<uint32_t> asks, result, meta(std::max<uint32_t>(nA, 1)), shp(meta.size()), sig(meta.size());
    std::vector<ykun::Segment> segs;
    yk::Orderer::Snap snap;
    yk_stats_t st{};
    const std::vector<uint8_t> npresent(nN, 1);
    const yklt::ChoiceIn in{o, ct, pending, nN, npresent.data(), n_total, nN, n_rank, nullptr, nullptr, !g_auto, automatic,
                            g_binpacking != 0, g_un_min, g_rd_min >= 0 ? g_rd_min : yklt::RD_MIN, scan, batch, g_auto ? nA : batch,
                            max_bindings, a_shape.data(), a_sigid.data(), asks, snap, meta.data(), shp.data(), sig.data(), segs, st};
    yklt::Choice choice;
    if (!yklt::choose_commit(in, choice)) return -1;
    if (!choice.device) return g_auto ? HOST_COMMIT : INELIGIBLE;

    // ---- device state: node records and the order (what yk_key_kernel + the radix sort + yk_lt_init_kernel build) ----
    const int RS = yklt::record_words(D);
    std::vector<int64_t> rec((size_t)std::max<uint32_t>(nN, 1) * RS, 0);
    std::vector<yklt::Ent> ord0(std::max<uint32_t>(nN, 1)), ord1(ord0.size());
    auto ent_lt = [](const yklt::Ent& x, const yklt::Ent& y) { return yklt::ent_less(x.key, x.rn, y.key, y.rn); };
    {
        std::vector<yklt::Ent> keys(nN);
        for (uint32_t n = 0; n < nN; ++n) {
            keys[n].key = yk_key_bits(yk_node_score(D, policy, weights, n_total + n, n_avail + n, nN));
            keys[n].rn = ((uint64_t)n_rank[n] << 32) | n;
            if (keys[n].key == YK_KEY_NAN) return -5;
        }
        std::sort(keys.begin(), keys.end(), ent_lt);
        std::vector<uint64_t> skey(nN);
        std::vector<uint32_t> snode(nN);
        for (uint32_t p = 0; p < nN; ++p) { skey[p] = keys[p].key; snode[p] = (uint32_t)keys[p].rn; }
        for (uint32_t p = 0; p < nN; ++p)
            yklt::init_node(D, (int)p, n_total, n_avail, nN, n_taint, n_label, n_flags, n_rank, skey.data(), snode.data(), rec.data(), RS,
                            ord0.data());
    }
    int cur = 0;
    int hdr[yklt::H_WORDS] = {0, 0, 0, 0, 0, 0, 0, 0};
    int64_t ub[8];
    for (int k = 0; k < 8; ++k) ub[k] = INT64_MAX;
    std::unique_ptr<yklt::Shared<D>> sh(new yklt::Shared<D>());

    yklt::Args la{};
    la.policy = policy;
    for (int k = 0; k < 8; ++k) la.w[k] = k < D ? weights[k] : 0.0;
    la.rec = rec.data(); la.RS = RS; la.ord[0] = ord0.data(); la.ord[1] = ord1.data(); la.cur = &cur; la.nlive = (int)nN;
    la.a_req = a_req; la.lda = nA; la.a_tol = a_tol; la.a_need = a_need; la.a_deny = a_deny; la.a_node = a_node;
    la.hdr = hdr; la.ub = ub; la.insensitive = ins ? 1 : 0;

    // the order must stay exactly: every node once, ascending by (CURRENT key, rank)
    auto order_ok = [&]() -> bool {
        const yklt::Ent* e = la.ord[cur];
        std::vector<uint8_t> seen(nN, 0);
        for (uint32_t p = 0; p < nN; ++p) {
            const uint32_t n = (uint32_t)e[p].rn;
            if (n >= nN || seen[n]) return false;
            seen[n] = 1;
            const int64_t* r = rec.data() + (size_t)n * RS;
            if (e[p].key != yk_key_bits(yk_node_score(D, policy, weights, r + D, r, 1)) || (e[p].rn >> 32) != n_rank[n]) return false;
            if (p > 0 && !ent_lt(e[p - 1], e[p])) return false;
        }
        return true;
    };
    // plain sequential first fit on the current order (stands in for the engine's host commit after a hand-off)
    auto resort = [&]() {
        yklt::Ent* e = la.ord[cur];
        for (uint32_t p = 0; p < nN; ++p) {
            const int64_t* r = rec.data() + (size_t)(uint32_t)e[p].rn * RS;
            e[p].key = yk_key_bits(yk_node_score(D, policy, weights, r + D, r, 1));
        }
        std::sort(e, e + nN, ent_lt);
    };
    auto seq_place = [&](uint32_t ask) -> uint32_t {
        int64_t rq[D];
        for (int k = 0; k < D; ++k) rq[k] = a_req[(size_t)k * nA + ask];
        const yklt::Ent* e = la.ord[cur];
        for (uint32_t p = 0; p < nN; ++p) {
            const uint32_t n = (uint32_t)e[p].rn;
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

    // a uniform run: the engine's attempt loop (ykun::uniform_run) with the kernels of yk_uniform.cuh replaced by loops over
    // the same per-item bodies -- lt_uniform's choice: a binpacking fill (un_fill) or a depth attempt (un_attempt)
    uint64_t attempts = 0;
    std::vector<uint32_t> byrank(nN);   // the nodes by ascending (NodeID rank, index)
    for (uint32_t i = 0; i < nN; ++i) byrank[i] = i;
    std::sort(byrank.begin(), byrank.end(), [&](uint32_t x, uint32_t y) { return n_rank[x] != n_rank[y] ? n_rank[x] < n_rank[y] : x < y; });
    auto uniform = [&](size_t off, size_t R, bool has_gang, int* ust, size_t* consumed) -> int {
        const int nlive = (int)nN;
        std::vector<uint32_t> cnt((size_t)nN, 0);
        std::vector<unsigned long long> bk((size_t)nlive), rkey((size_t)nlive), rrn((size_t)nlive), okey((size_t)nlive), orn((size_t)nlive);
        const uint32_t ask = asks[off];
        ykun::Args a{};
        a.policy = la.policy;
        for (int k = 0; k < 8; ++k) { a.w[k] = la.w[k]; a.req[k] = k < D ? la.a_req[(size_t)k * la.lda + ask] : 0; }
        a.rec = la.rec; a.RS = la.RS; a.ord[0] = la.ord[0]; a.ord[1] = la.ord[1]; a.cur = la.cur; a.nlive = nlive; a.byrank = byrank.data();
        a.tol = la.a_tol[ask]; a.need = la.a_need[ask]; a.deny = la.a_deny[ask]; a.want = la.a_node[ask];
        a.R = (int)R; a.insensitive = la.insensitive; a.has_gang = has_gang ? 1 : 0;
        a.bk = bk.data(); a.cnt = cnt.data(); a.rkey = rkey.data(); a.rrn = rrn.data(); a.okey = okey.data(); a.orn = orn.data();
        a.res = result.data() + off;
        auto attempt = [&](int L, ykun::Globals& g) -> int {
            a.L = L; a.g = &g;
            const size_t ne = (size_t)nlive * (size_t)L;
            std::vector<unsigned long long> ekey(ne), skey(ne);
            std::vector<uint32_t> enode(ne), snode(ne), idx(ne);
            a.ekey = ekey.data(); a.enode = enode.data(); a.skey = skey.data(); a.snode = snode.data();
            g.bkey = ykun::KEY_INF; g.brank = ykun::KEY_INF; g.last_key = 0; g.last_rank = 0; g.valid = 0; g.nan = 0; g.status = ykun::U_RETRY; g.consumed = 0;
            for (long long x = 0; x < (long long)ne; ++x) {
                const ykun::DepthOut o = ykun::element_item<D>(a, x);
                g.valid += o.valid;
                if (o.bk < g.bkey) g.bkey = o.bk;
                if (o.nan) g.nan = 1;
            }
            if (!bp)
                for (int i = 0; i < nlive; ++i) { const unsigned long long r = ykun::brank_item<D>(a, i, g.bkey); if (r < g.brank) g.brank = r; }
            for (size_t x = 0; x < ne; ++x) idx[x] = (uint32_t)x;
            std::stable_sort(idx.begin(), idx.end(), [&](uint32_t x, uint32_t y) { return ekey[x] < ekey[y]; });
            for (size_t x = 0; x < ne; ++x) { skey[x] = ekey[idx[x]]; snode[x] = enode[idx[x]]; }
            if (bp) {   // capacities clamped to R, their inclusive sum, then one search per ask
                unsigned long long sum = 0;
                for (int p = 0; p < nlive; ++p) { ykun::fill_cap_item<D>(a, p); sum += ekey[(size_t)p]; bk[(size_t)p] = sum; }
                ykun::fill_decide(a);
                for (int q = 0; q < (int)R; ++q) ykun::fill_select_item(a, q, g.valid);
            } else {
                for (int q = 0; q < (int)R; ++q) ykun::select_item<D>(a, q, g.valid);
                ykun::decide(a);
            }
            for (int i = 0; i < nlive; ++i) { ykun::apply_item<D>(a, i, g.status); if (ykun::rekey_item<D>(a, i)) g.nan = 2; }
            {   // the order after the run (what un_reorder builds from the re-keyed entries)
                std::vector<uint32_t> ix((size_t)nlive);
                for (int i = 0; i < nlive; ++i) ix[(size_t)i] = (uint32_t)i;
                std::stable_sort(ix.begin(), ix.end(), [&](uint32_t x, uint32_t y) { return rkey[x] < rkey[y]; });
                yklt::Ent* e = la.ord[*la.cur & 1];
                for (int p = 0; p < nlive; ++p) { e[p].key = rkey[ix[(size_t)p]]; e[p].rn = rrn[ix[(size_t)p]]; }
            }
            for (uint32_t c : cnt) if (c) return -99;   // counters must be clean after every attempt
            ++attempts;
            return 0;
        };
        const int rc = ykun::uniform_run(D, la.w, a.req, n_total, nN, byrank.data(), nlive, (int)R, g_un_depth, st, attempt, ust, consumed, bp);
        if (rc) return rc;
        return *ust == ykun::U_NAN || order_ok() ? 0 : -9;
    };
    // a stretch on the lattice kernel: yk_lattice_kernel's body as plain loops
    auto window = [&](size_t off, size_t len, int* status, size_t* consumed) -> int {
        la.asks = asks.data() + off; la.meta = meta.data() + off; la.shp = shp.data() + off; la.sig = sig.data() + off;
        la.B = (int)len; la.res = result.data() + off;
        yklt::lattice_batch<D>(la, *sh);
        *status = hdr[yklt::H_STATUS];
        *consumed = (size_t)hdr[yklt::H_CONSUMED];
        return *status == yklt::ST_NAN || order_ok() ? 0 : -9;
    };
    // a round-eligible stretch: yk_rounds_kernel's body as plain loops
    std::vector<yklt::Ent> spent(std::max<uint32_t>(nN, 1));
    std::unique_ptr<ykrd::Shared> rs(new ykrd::Shared());
    int rhdr[ykrd::R_WORDS] = {0, 0, 0, 0, 0};
    uint64_t passes = 0, singles = 0, round_asks = 0, round_stretches = 0, parked = 0;
    auto rounds = [&](size_t off, size_t len, int* status, size_t* consumed) -> int {
        ykrd::Args ra{};
        ra.policy = la.policy;
        for (int k = 0; k < 8; ++k) ra.w[k] = la.w[k];
        ra.rec = la.rec; ra.RS = RS; ra.ord[0] = la.ord[0]; ra.ord[1] = la.ord[1]; ra.cur = la.cur; ra.nlive = (int)nN; ra.spent = spent.data();
        ra.a_req = a_req; ra.lda = nA; ra.a_tol = a_tol; ra.a_need = a_need; ra.a_deny = a_deny; ra.a_node = a_node;
        ra.asks = asks.data() + off; ra.B = (int)len; ra.res = result.data() + off; ra.hdr = rhdr;
        ra.window = g_rd_window > 0 ? std::min(g_rd_window, ykrd::WCAP) : ykrd::WCAP;
        ra.guard = g_rd_guard >= 0 ? g_rd_guard : ykrd::GUARD;
        ykrd::rounds_stretch<D>(ra, *rs);
        *status = rhdr[ykrd::R_STATUS];
        *consumed = (size_t)rhdr[ykrd::R_CONSUMED];
        passes += (uint64_t)rhdr[ykrd::R_PASSES]; parked += (uint64_t)rhdr[ykrd::R_SPENT]; singles += (uint64_t)rhdr[ykrd::R_SINGLES]; round_asks += *consumed; ++round_stretches;
        return *status == yklt::ST_NAN || order_ok() ? 0 : -9;
    };
    auto device_batch = [&](size_t B, int* status, size_t* consumed) -> int {
        result.assign(B, yk::CNONE);
        return yklt::route_batch(bp, g_auto || g_rounds != 0, ct, ins, taints, asks.data(), segs, meta.data(), uniform, rounds, window, status, consumed);
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

    bool handoff = false;
    yklt::Loop lp{o, ct, choice.shape_ids, a_sigid.data(), asks, snap, result, meta.data(), shp.data(), sig.data(), segs,
                  choice.plan_ready, yklt::min_run(bp, g_un_min), nN == 0, ins ? (size_t)in.maxA : batch, max_bindings, n, st};
    int rc = yklt::device_commit(lp, device_batch, bind, fail, handoff);
    if (!rc && handoff) {   // the engine's path: the rest of the cycle on the host commit, never back on the device
        lp.min_run = 0;
        size_t bsz = batch;
        if (!yk::fill_batch(o, bsz, batch, (size_t)max_bindings - n, asks, snap, st)) return -1;
        rc = yklt::device_commit(lp, sequential, bind, fail, handoff);
    }
    if (rc) return rc;
    o.finish();
    *n_out = n;
    for (uint32_t i = 0; i < nA; ++i) state_out[i] = tb.state[i];
    for (uint32_t nn = 0; nn < nN; ++nn)
        for (int k = 0; k < D; ++k) avail_out[(size_t)k * nN + nn] = rec[(size_t)nn * RS + k];
    if (stats_out) {   // one layout for every mode, read by name (tests/device_shim.py STATS); a word a mode never touches stays 0
        const uint64_t c[] = {(uint64_t)hdr[yklt::H_SUBRUNS], (uint64_t)hdr[yklt::H_FULLSCANS], (uint64_t)hdr[yklt::H_SORTS],
                              (uint64_t)hdr[yklt::H_ELEMS], (uint64_t)hdr[yklt::H_QUICK], (uint64_t)hdr[yklt::H_ESC],
                              st.lattice_handoffs, st.batches, attempts, st.uniform_retries, st.uniform_asks, st.uniform_runs,
                              st.uniform_elements, passes, singles, round_asks, round_stretches, parked, 1};
        std::copy(c, c + sizeof(c) / sizeof(c[0]), stats_out);
    }
    return 0;
}

}  // namespace

// same argument list as engine_host_run (tests/host/engine_shim.cpp) so that the Python harness is shared; epoch_limit,
// speculate and share_rows do not apply.  Returns INELIGIBLE when the snapshot is not eligible for the forced device
// commit, HOST_COMMIT when `auto` starts the cycle on the host commit.
extern "C" int device_host_run(int D, uint32_t policy, const double* weights,
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

// ykun::plan_segments / cap_of_d / first_depth for the unit tests
extern "C" int host_plan_segments(const uint32_t* meta, const uint32_t* shp, const uint32_t* sig, int B, int min_run, int* off, int* len, int* uniform, int cap) {
    std::vector<ykun::Segment> segs;
    ykun::plan_segments(meta, shp, sig, B, min_run, segs);
    int n = 0;
    for (const ykun::Segment& s : segs) { if (n < cap) { off[n] = s.off; len[n] = s.len; uniform[n] = s.uniform ? 1 : 0; } ++n; }
    return n;
}
extern "C" int64_t host_cap_of(int D, int usable, const int64_t* avail, const int64_t* total, const int64_t* req, int64_t limit) {
    return ykun::cap_of_d(D, usable != 0, avail, total, req, limit);
}
extern "C" int host_first_depth(int R, int nlive) { return ykun::first_depth(R, nlive); }
