// Host-only emulation of yk_cycle for the CPU test suite: the REAL ordering engine (csrc/yk_orderer.hpp) and the REAL
// ordered commit (csrc/yk_commit.hpp: epochs, touched-node index, gang roll-back, order merge) driven by the engine's own
// batch loop (yk::host_commit in csrc/yk_lattice_host.hpp: two slots, speculative next batch, rewind, epoch ends) -- only
// the device part is replaced: the fit rows are computed here by a plain CPU loop over the epoch's sorted view, and the
// speculated fill runs inline (test infrastructure, never part of the product).  What this cannot cover is the CUDA
// kernels, the stream plumbing and the helper thread: those are the `-m gpu` tests.
#include "../../yunikorn_k8shim_b200/csrc/yk_lattice_host.hpp"
#include "shim_tables.hpp"

#include <algorithm>
#include <cstdint>
#include <thread>
#include <vector>
#if defined(__x86_64__)
#include <immintrin.h>
#endif

// ---- bench arm "cpu_engine" (bench.py): the same orderer + ordered commit with the sweep done by the host cores ----
// g_sweep_threads == 0: the plain scalar test loop below (what the CPU test suite runs).  > 0: rows are swept by that many
// threads, eight sorted positions per AVX-512 compare when the CPU has it (a column-major copy of the epoch view is kept
// for it) -- the honest "no GPU" version of this engine, timed next to the GPU one.  g_skip_checks drops the O(N)
// self-checks the test harness runs after every epoch.
static int g_sweep_threads = 0;
static int g_skip_checks = 0;
extern "C" void host_set_bench_mode(int threads, int skip_checks) { g_sweep_threads = threads; g_skip_checks = skip_checks; }

namespace {
static int g_profile = 0;
extern "C" void host_set_profile(int on) { g_profile = on; }

struct SoAView { const int64_t* cap; size_t ld; const uint64_t* taint; const uint64_t* label; const uint32_t* node; int D; int Np; };

void sweep_row_scalar(const SoAView& v, const int64_t* rq, uint64_t tol, uint64_t need, uint64_t deny, uint32_t want, uint32_t* row, int W) {
    row[W] = yk::CNONE;
    for (int p = 0; p < v.Np; ++p) {
        bool ok = true;
        for (int k = 0; k < v.D; ++k) ok = ok && rq[k] <= v.cap[(size_t)k * v.ld + p];
        ok = ok && !((v.taint[p] & ~tol) | (~v.label[p] & need) | (v.label[p] & deny));
        ok = ok && (want == yk::CNONE || want == v.node[p]);
        if (ok) { row[p >> 5] |= 1u << (p & 31); if (row[W] == yk::CNONE) row[W] = (uint32_t)p; }
    }
}

#if defined(__x86_64__)
__attribute__((target("avx512f,avx512bw,avx512vl")))
void sweep_row_avx512(const SoAView& v, const int64_t* rq, uint64_t tol, uint64_t need, uint64_t deny, uint32_t want, uint32_t* row, int W) {
    row[W] = yk::CNONE;
    const __m512i ntol = _mm512_set1_epi64((long long)~tol), vneed = _mm512_set1_epi64((long long)need), vdeny = _mm512_set1_epi64((long long)deny);
    const __m512i vwant = _mm512_set1_epi64((long long)want);
    __m512i r[8];
    for (int k = 0; k < v.D; ++k) r[k] = _mm512_set1_epi64(rq[k]);
    for (int w = 0; w < W; ++w) {
        uint32_t bits = 0;
        for (int q = 0; q < 4; ++q) {
            const int p = w * 32 + q * 8;
            __mmask8 m = 0xFF;
            for (int k = 0; k < v.D; ++k) m &= _mm512_cmple_epi64_mask(r[k], _mm512_loadu_si512(v.cap + (size_t)k * v.ld + p));
            const __m512i t = _mm512_loadu_si512(v.taint + p), l = _mm512_loadu_si512(v.label + p);
            m &= _mm512_testn_epi64_mask(t, ntol);                                   // (taint & ~tol) == 0
            m &= _mm512_cmpeq_epi64_mask(_mm512_and_si512(l, vneed), vneed);          // (label & need) == need
            m &= _mm512_testn_epi64_mask(l, vdeny);                                   // (label & deny) == 0
            if (want != yk::CNONE) m &= _mm512_cmpeq_epi64_mask(_mm512_cvtepu32_epi64(_mm256_loadu_si256((const __m256i*)(v.node + p))), vwant);
            bits |= (uint32_t)m << (q * 8);
        }
        row[w] = bits;
        if (bits && row[W] == yk::CNONE) row[W] = (uint32_t)w * 32u + (uint32_t)__builtin_ctz(bits);
    }
}
#endif
}  // namespace


namespace {
struct Slot { std::vector<uint32_t> asks, reps, row_of; yk::Orderer::Snap snap; std::vector<uint32_t> fit; };
}

// exchange callback with the signature of yk_allgather_fn (include/ykgpu.h): all-gather of equal row blocks, in place
typedef int (*shim_allgather_fn)(void* ctx, void* buf, uint64_t row_bytes, uint32_t first_row, uint32_t n_rows, uint32_t total_rows, void* stream);

static int engine_host_run_impl(
    uint32_t rank, uint32_t world, shim_allgather_fn xfn, uint64_t split_min_pairs,
    int D, uint32_t policy, const double* weights,
    uint32_t nN, const int64_t* n_total /*[D][nN]*/, const int64_t* n_avail, const uint64_t* n_taint, const uint64_t* n_label,
    const uint32_t* n_flags, const uint32_t* n_rank,
    uint32_t nA, uint32_t nP, uint32_t nQ, const int64_t* a_req /*[D][nA]*/, const uint64_t* a_tol, const uint64_t* a_need,
    const uint64_t* a_deny, const uint32_t* a_node, const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app,
    const uint32_t* a_flags, const uint32_t* a_gang, const uint32_t* p_queue, const int64_t* p_submit,
    const uint32_t* q_parent, const int64_t* q_guar, const int64_t* q_max, int64_t* q_alloc, const uint8_t* q_sort,
    uint32_t batch, uint32_t epoch_limit, int speculate, int share_rows, uint32_t max_bindings,
    uint32_t* out_ask, uint32_t* out_node, uint32_t* n_out, uint8_t* state_out, int64_t* avail_out /*[D][nN]*/, uint64_t* rows_out) {
    // ---- orderer ----
    yk::Orderer o;
    ShimTables tb;
    wire_orderer(o.t, tb, D, nA, nP, nQ, a_req, a_prio, a_create, a_app, a_flags, a_gang, p_queue, p_submit, q_parent, q_guar, q_max,
                 q_alloc, q_sort);
    std::vector<uint32_t> pending(nA);
    for (uint32_t i = 0; i < nA; ++i) pending[i] = i;
    o.begin_cycle(pending);
    const bool ins = o.insensitive;

    // ---- committer + initial order (what yk_key_kernel + the stable radix sort produce) ----
    yk::Committer cm;
    cm.profile = g_profile != 0;
    cm.t.D = D; cm.t.policy = policy; cm.t.w = weights; cm.t.lda = nA;
    cm.t.a_req = a_req; cm.t.a_tol = a_tol; cm.t.a_need = a_need; cm.t.a_deny = a_deny; cm.t.a_node = a_node; cm.t.a_gang = a_gang; cm.t.a_app = a_app;
    cm.build(nN, n_avail, n_total, nN, n_taint, n_label, n_rank);
    cm.set_pending(pending);
    const int nlive = (int)nN;
    std::vector<uint32_t> order_nodes(nN);   // what the engine uploads for the device's gather
    {
        std::vector<yk::DirtyRef> ks(nN);
        for (uint32_t n = 0; n < nN; ++n) {
            const double sc = yk_node_score(D, policy, weights, n_total + n, n_avail + n, nN);
            ks[n] = yk::DirtyRef(yk_key_bits(sc), n_rank[n], n);
        }
        std::sort(ks.begin(), ks.end());
        std::vector<uint64_t> keys(nN);
        for (uint32_t p = 0; p < nN; ++p) { order_nodes[p] = ks[p].node(); keys[p] = ks[p].key(); }
        cm.set_order(order_nodes.data(), keys.data(), nlive);
    }
    // ---- the epoch's sorted view (what yk_gather_kernel builds) and the CPU stand-in for the sweep ----
    const int W = nlive ? (nlive + 511) / 512 * 16 : 0;   // same rounding as the engine: tiles of 512 positions
    const int WS = W + 1;
    std::vector<int64_t> v_cap;   // [pos][D]
    std::vector<int64_t> v_capT;  // [D][pos]: the column-major copy the vectorised bench sweep reads
    std::vector<uint64_t> v_taint, v_label;
    std::vector<uint32_t> v_node;
    auto refresh_view = [&]() {
        v_cap.assign((size_t)W * 32 * D, -1); v_taint.assign((size_t)W * 32, ~0ull); v_label.assign((size_t)W * 32, 0); v_node.assign((size_t)W * 32, yk::CNONE);
        for (int p = 0; p < nlive; ++p) {
            const uint32_t n = order_nodes[p];
            const bool usable = (n_flags[n] & 1u) && !(n_flags[n] & 2u);
            yk::NodeView nv = cm.node(n);
            for (int k = 0; k < D; ++k) {   // same fold as yk_gather_kernel, from the commit's current availability
                const int64_t a = std::max<int64_t>(0, nv.avail()[k]), t = std::max<int64_t>(0, nv.total()[k]);
                v_cap[(size_t)p * D + k] = usable ? std::min(a, t) : -1;
            }
            v_taint[p] = n_taint[n]; v_label[p] = n_label[n]; v_node[p] = n;
        }
        if (g_sweep_threads > 0) {
            const size_t Np = (size_t)W * 32;
            v_capT.resize(Np * D);
            for (size_t p = 0; p < Np; ++p) for (int k = 0; k < D; ++k) v_capT[(size_t)k * Np + p] = v_cap[p * D + k];
        }
        cm.begin_epoch(W);
    };
    std::vector<uint64_t> a_sig(nA);
    // the engine does this in yk_asks_upsert; share_rows == 2 makes every hash collide (equality must come from the full compare)
    for (uint32_t a = 0; a < nA; ++a) a_sig[a] = share_rows == 2 ? 42 : yk::ask_signature(cm.t, a);
    yk::RowShare share;
    uint64_t rows_swept = 0;
    int xrc = 0;
    auto sweep = [&](Slot& sl) {
        if (sl.asks.empty()) { sl.reps.clear(); sl.row_of.clear(); sl.fit.clear(); return; }   // produce() returns early as well
        share.build(cm.t, a_sig.data(), sl.asks, share_rows != 0, sl.reps, sl.row_of);   // as produce() does
        rows_swept += sl.reps.size();
        // this rank's shard of the rows, exactly as produce() cuts it (world == 1 or a small sweep: all of them)
        const size_t R = sl.reps.size();
        const bool split = world > 1 && (uint64_t)R * (uint64_t)nlive >= split_min_pairs;
        const size_t G = split ? world : 1, my = split ? rank : 0;
        const size_t rows_per = (R + G - 1) / G, row0 = std::min(R, my * rows_per), row1 = std::min(R, row0 + rows_per);
        sl.fit.assign(rows_per * G * (size_t)WS, 0);
        if (g_sweep_threads > 0) {   // bench arm: every row by the host cores, vectorised
            const SoAView view{v_capT.data(), (size_t)W * 32, v_taint.data(), v_label.data(), v_node.data(), D, W * 32};
#if defined(__x86_64__)
            const bool avx = __builtin_cpu_supports("avx512f") && __builtin_cpu_supports("avx512bw");
#else
            const bool avx = false;
#endif
            auto work = [&](size_t lo, size_t hi) {
                for (size_t i = lo; i < hi; ++i) {
                    const uint32_t a = sl.reps[i];
                    int64_t rq[8];
                    for (int k = 0; k < D; ++k) rq[k] = a_req[(size_t)k * nA + a];
                    uint32_t* row = sl.fit.data() + i * WS;
#if defined(__x86_64__)
                    if (avx) { sweep_row_avx512(view, rq, a_tol[a], a_need[a], a_deny[a], a_node[a], row, W); continue; }
#endif
                    sweep_row_scalar(view, rq, a_tol[a], a_need[a], a_deny[a], a_node[a], row, W);
                }
            };
            const size_t nr = row1 - row0;
            const size_t T = std::max<size_t>(1, std::min<size_t>((size_t)g_sweep_threads, nr / 64));
            if (T <= 1) work(row0, row1);
            else {
                std::vector<std::thread> th;
                for (size_t x = 0; x < T; ++x) th.emplace_back(work, row0 + nr * x / T, row0 + nr * (x + 1) / T);
                for (auto& t : th) t.join();
            }
        } else
        for (size_t i = row0; i < row1; ++i) {
            const uint32_t a = sl.reps[i];
            uint32_t* row = sl.fit.data() + i * WS;
            row[W] = yk::CNONE;
            for (int p = 0; p < W * 32; ++p) {
                bool ok = true;
                for (int k = 0; k < D; ++k) ok = ok && a_req[(size_t)k * nA + a] <= v_cap[(size_t)p * D + k];
                ok = ok && !((v_taint[p] & ~a_tol[a]) | (~v_label[p] & a_need[a]) | (v_label[p] & a_deny[a]));
                ok = ok && (a_node[a] == yk::CNONE || a_node[a] == v_node[p]);
                if (ok) { row[p >> 5] |= 1u << (p & 31); if (row[W] == yk::CNONE) row[W] = (uint32_t)p; }
            }
        }
        if (split) {   // the other ranks' rows arrive through the exchange callback (the engine's yk_set_exchange path)
            if (!xfn || xfn(nullptr, sl.fit.data(), (uint64_t)WS * 4, (uint32_t)row0, (uint32_t)rows_per, (uint32_t)(rows_per * G), nullptr) != 0) xrc = -11;
        }
    };
    refresh_view();
    // the epoch ends: merge the order, check it (unless g_skip_checks) and refresh the view
    auto new_epoch = [&]() -> int {
        if (!cm.dirty_list.empty()) {
            cm.merge_order(order_nodes.data(), nlive);
            if (!g_skip_checks) {   // the merged order must be exactly: every node once, ascending by (CURRENT score key, NodeID rank)
                std::vector<uint8_t> seen_node(nN, 0);
                for (int p = 0; p < nlive; ++p) {
                    const yk::DirtyRef r = cm.order()[p];
                    const uint32_t nn = r.node();
                    if (nn >= nN || seen_node[nn] || order_nodes[p] != nn) return -7;
                    seen_node[nn] = 1;
                    yk::NodeView nv = cm.node(nn);
                    const double sc = yk_node_score(D, policy, weights, nv.total(), nv.avail(), 1);
                    if (r.key() != yk_key_bits(sc) || r.rank() != n_rank[nn]) return -8;
                    if (p > 0 && !(cm.order()[p - 1] < r)) return -9;
                }
            }
        }
        refresh_view();
        return 0;
    };

    // ---- the engine's batch loop (yk::host_commit), speculated fills run inline ----
    Slot slot[2];
    uint32_t n = 0;
    std::vector<uint32_t> result;
    yk_stats_t st{};
    size_t bsz = batch;
    if (!yk::fill_batch(o, bsz, batch, max_bindings, slot[0].asks, slot[0].snap, st)) return -1;
    yk::HostLoop lp{o, result, nlive == 0, batch, epoch_limit, cm.dirty_list, speculate != 0, max_bindings, n, st, st};
    const int rc = yk::host_commit(lp, slot,
                                   [&](Slot& sl, yk_stats_t&) { sweep(sl); return xrc; },
                                   [&](Slot& sl, std::vector<uint32_t>& res, size_t& consumed) {
                                       return cm.commit_batch(sl.asks, sl.row_of.data(), sl.fit.data(), ins, res, consumed,
                                                              [&](int) { return (int)sl.reps.size(); });
                                   },
                                   [](auto&& job) { job(); }, [] {}, [](Slot&) { return 0; }, new_epoch,
                                   [&](uint32_t a, uint32_t node) { out_ask[n] = a; out_node[n] = node; ++n; },
                                   [](int, const char*) { return -1; });   // the loop's own error: a gang no batch holds
    if (rc) return rc;
    o.finish();
    *n_out = n;
    if (rows_out) {   // [0] rows swept, then the commit's counters (yk_commit.hpp dbg[]: words scanned, touched candidates walked,
        rows_out[0] = rows_swept;   // asks won by a touched node, re-keys) and its TSC profile when host_set_profile(1) was called
        for (int k = 0; k < 4; ++k) rows_out[1 + k] = cm.dbg[k];
        for (int k = 0; k < 6; ++k) rows_out[5 + k] = cm.prof[k];
    }
    for (uint32_t i = 0; i < nA; ++i) state_out[i] = tb.state[i];
    for (uint32_t nn = 0; nn < nN; ++nn)
        for (int k = 0; k < D; ++k) avail_out[(size_t)k * nN + nn] = cm.node(nn).avail()[k];
    return 0;
}

extern "C" int engine_host_run(int D, uint32_t policy, const double* weights,
    uint32_t nN, const int64_t* n_total /*[D][nN]*/, const int64_t* n_avail, const uint64_t* n_taint, const uint64_t* n_label,
    const uint32_t* n_flags, const uint32_t* n_rank,
    uint32_t nA, uint32_t nP, uint32_t nQ, const int64_t* a_req /*[D][nA]*/, const uint64_t* a_tol, const uint64_t* a_need,
    const uint64_t* a_deny, const uint32_t* a_node, const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app,
    const uint32_t* a_flags, const uint32_t* a_gang, const uint32_t* p_queue, const int64_t* p_submit,
    const uint32_t* q_parent, const int64_t* q_guar, const int64_t* q_max, int64_t* q_alloc, const uint8_t* q_sort,
    uint32_t batch, uint32_t epoch_limit, int speculate, int share_rows, uint32_t max_bindings,
    uint32_t* out_ask, uint32_t* out_node, uint32_t* n_out, uint8_t* state_out, int64_t* avail_out /*[D][nN]*/, uint64_t* rows_out) {
    return engine_host_run_impl(0, 1, nullptr, 0, D, policy, weights, nN, n_total, n_avail, n_taint, n_label, n_flags, n_rank, nA, nP, nQ, a_req, a_tol, a_need, a_deny, a_node, a_prio, a_create, a_app, a_flags, a_gang, p_queue, p_submit, q_parent, q_guar, q_max, q_alloc, q_sort, batch, epoch_limit, speculate, share_rows, max_bindings, out_ask, out_node, n_out, state_out, avail_out, rows_out);
}

// the same cycle as one of `world` replicas: rows of each batch are cut across the ranks and exchanged through xfn
extern "C" int engine_host_run_ranked(uint32_t rank, uint32_t world, shim_allgather_fn xfn, uint64_t split_min_pairs, int D, uint32_t policy, const double* weights,
    uint32_t nN, const int64_t* n_total /*[D][nN]*/, const int64_t* n_avail, const uint64_t* n_taint, const uint64_t* n_label,
    const uint32_t* n_flags, const uint32_t* n_rank,
    uint32_t nA, uint32_t nP, uint32_t nQ, const int64_t* a_req /*[D][nA]*/, const uint64_t* a_tol, const uint64_t* a_need,
    const uint64_t* a_deny, const uint32_t* a_node, const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app,
    const uint32_t* a_flags, const uint32_t* a_gang, const uint32_t* p_queue, const int64_t* p_submit,
    const uint32_t* q_parent, const int64_t* q_guar, const int64_t* q_max, int64_t* q_alloc, const uint8_t* q_sort,
    uint32_t batch, uint32_t epoch_limit, int speculate, int share_rows, uint32_t max_bindings,
    uint32_t* out_ask, uint32_t* out_node, uint32_t* n_out, uint8_t* state_out, int64_t* avail_out /*[D][nN]*/, uint64_t* rows_out) {
    return engine_host_run_impl(rank, world, xfn, split_min_pairs, D, policy, weights, nN, n_total, n_avail, n_taint, n_label, n_flags, n_rank, nA, nP, nQ, a_req, a_tol, a_need, a_deny, a_node, a_prio, a_create, a_app, a_flags, a_gang, p_queue, p_submit, q_parent, q_guar, q_max, q_alloc, q_sort, batch, epoch_limit, speculate, share_rows, max_bindings, out_ask, out_node, n_out, state_out, avail_out, rows_out);
}

// csrc/yk_score.h compiled for the host (the same code the device runs): for the score known-answer test
extern "C" double score_host(int D, uint32_t policy, const double* w, const int64_t* total, const int64_t* avail) {
    return yk_node_score(D, policy, w, total, avail, 1);
}
