// yk_engine.cu -- libykgpu.so: host side of the engine + the C ABI of include/ykgpu.h.
//
// One scheduling cycle (yk_cycle) =
//   host  : Orderer (yk_orderer.hpp) produces the next batch of asks in schedule()-pass order
//   device: key kernel (float64 node score) -> stable radix sort by key over NodeID-rank order
//           -> gather into the sorted SoA view -> fused sweep kernel (batch x all nodes) -> fit bitmaps
//   commit: ordered, exact: ask i takes the minimum (key, NodeID) over {clean nodes whose bitmap bit is set}
//           U {nodes already committed to in this batch, re-scored}; see DESIGN.md "ordered commit".
// There is no CPU fallback for the sweep: without a CUDA device yk_create fails with YK_ERR_CUDA.
#include "../../include/ykgpu.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <thread>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <mutex>
#include <new>
#include <string>
#include <vector>
#include <x86intrin.h>

#include "yk_kernels.cuh"
#include "yk_filter.cuh"
#include "yk_preempt_nodes.cuh"
#include "yk_preempt_plan.cuh"
#include "yk_preempt_required.cuh"
#include "yk_lattice.cuh"
#include "yk_uniform.cuh"
#include "yk_rounds.cuh"
#include "yk_spec.cuh"
#include "yk_commit.hpp"
#include "yk_lattice_host.hpp"
#include "yk_orderer.hpp"

namespace {

#ifndef YK_NPT
#define YK_NPT 2
#endif
constexpr int NPT = YK_NPT;       // sorted-node positions per sweep thread
constexpr int AC = 128;           // asks per sweep CTA chunk
constexpr int NODE_TILE = YK_SWEEP_THREADS * NPT;

inline size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }

template <typename T>
struct Dev {
    T* p = nullptr; size_t n = 0;
    cudaError_t alloc(size_t count) {
        free();
        n = count;
        return cudaMalloc((void**)&p, std::max<size_t>(count, 1) * sizeof(T));
    }
    void free() { if (p) cudaFree(p); p = nullptr; n = 0; }
    ~Dev() { free(); }
};
template <typename T>
struct Pin {
    T* p = nullptr; size_t n = 0;
    T* d = nullptr;   // alloc(count, true): the device's address of the same memory (mapped), which kernels write directly
    cudaError_t alloc(size_t count, bool mapped = false) {
        free();
        n = count;
        cudaError_t e = cudaHostAlloc((void**)&p, std::max<size_t>(count, 1) * sizeof(T), mapped ? cudaHostAllocMapped : cudaHostAllocDefault);
        if (e == cudaSuccess) memset(p, 0, std::max<size_t>(count, 1) * sizeof(T));
        if (e == cudaSuccess && mapped) e = cudaHostGetDevicePointer((void**)&d, p, 0);
        return e;
    }
    void free() { if (p) cudaFreeHost(p); p = nullptr; d = nullptr; n = 0; }
    T& operator[](size_t i) { return p[i]; }
    const T& operator[](size_t i) const { return p[i]; }
    ~Pin() { free(); }
};


double now_ms() {
    using namespace std::chrono;
    return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

// A helper thread that fills and launches the NEXT batch while the caller's thread commits the current one
// (the orderer state is only touched by one of the two at a time: fork before the commit, join after it).
struct Worker {
    std::thread th;
    std::mutex m;
    std::condition_variable cv;
    std::function<void()> job;
    bool has_job = false, busy = false, quit = false;
    int device = 0;
    void start(int dev) {
        device = dev;
        th = std::thread([this] {
            cudaSetDevice(device);
            std::unique_lock<std::mutex> lk(m);
            for (;;) {
                cv.wait(lk, [this] { return has_job || quit; });
                if (quit) return;
                has_job = false;
                lk.unlock();
                job();
                lk.lock();
                busy = false;
                cv.notify_all();
            }
        });
    }
    void submit(std::function<void()> f) {
        std::lock_guard<std::mutex> lk(m);
        job = std::move(f); has_job = true; busy = true;
        cv.notify_all();
    }
    void wait() {
        std::unique_lock<std::mutex> lk(m);
        cv.wait(lk, [this] { return !busy; });
    }
    void stop() {
        if (!th.joinable()) return;
        { std::lock_guard<std::mutex> lk(m); quit = true; cv.notify_all(); }
        th.join();
    }
};

// One in-flight batch: its asks, device / pinned buffers and read-back events.  Two slots let the sweep and the
// read-back of batch k+1 run while the host commits batch k (both against the same epoch view, see run loop).
struct Slot {
    std::vector<uint32_t> asks;     // the batch, in commit order
    std::vector<uint32_t> reps;     // one representative ask per distinct signature = the rows the device sweeps
    std::vector<uint32_t> row_of;   // batch entry -> row
    yk::Orderer::Snap snap;
    Dev<uint32_t> d_batch, d_fit;
    Pin<uint32_t> h_batch, h_fit;
    Pin<int> h_err;                 // P2P: copy of the device error word after the flag waits
    std::vector<cudaEvent_t> ev;
    cudaEvent_t ev_s0 = nullptr, ev_s1 = nullptr;
    int B = 0, R = 0, W = 0, chunk = 0, nchunks = 0, rows = 0;   // B asks, R rows (all ranks), rows = this rank's shard
    uint32_t last_value = 0;        // P2P: sequence value signalled when this slot's previous content was published
};

// Signature numbers, kept up to date as asks are upserted: equal number <=> equal predicate signature (request vector,
// tolerations, required / forbidden labels, node name).  Open addressing on the 64-bit signature hash; a hit is always
// confirmed on the full signature of the entry's representative ask.  (A representative that was later overwritten with
// another signature just stops matching: the signature then gets a second number -- an extra swept row, never a wrong
// merge.)  Rebuilt from the present asks when it has handed out more than four numbers per ask slot.
struct SigTable {
    struct Ent { uint64_t h; uint32_t rep, id; };
    static constexpr uint32_t FREE = 0xFFFFFFFFu, TOMB = 0xFFFFFFFEu;
    std::vector<Ent> tab;
    std::vector<uint32_t> rep_slot;   // ask -> 1 + the slot it represents, 0 when it represents none
    uint32_t n = 0;
    void reset(size_t asks) {
        size_t cap = 1024;
        while (cap < 4 * asks) cap <<= 1;
        tab.assign(cap, Ent{0, FREE, 0});
        rep_slot.assign(asks, 0);
        n = 0;
    }
    // the ask's row is about to be overwritten: a number it represents is never handed out again (the asks that hold it
    // stay equal among themselves; the signature gets a fresh number next time it is seen)
    void retire(uint32_t ask) {
        if (rep_slot[ask]) { tab[rep_slot[ask] - 1].rep = TOMB; rep_slot[ask] = 0; }
    }
    uint32_t get(const yk::CommitTables& t, uint64_t h, uint32_t ask) {
        const size_t mask = tab.size() - 1;
        size_t x = (size_t)(h ^ (h >> 29)) & mask;
        for (;;) {
            Ent& e = tab[x];
            if (e.rep == FREE) { e.h = h; e.rep = ask; e.id = n++; rep_slot[ask] = (uint32_t)x + 1; return e.id; }
            if (e.rep != TOMB && e.h == h && yk::same_signature(t, e.rep, ask)) return e.id;
            x = (x + 1) & mask;
        }
    }
};

}  // namespace

struct yk_engine {
    std::mutex mu;
    yk_config cfg{};
    int D = 0;
    uint32_t maxN = 0, maxA = 0, maxP = 0, maxQ = 0, batch = 0;
    std::string err;
    yk_stats_t st{};
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr;
    YkWeights w{};

    // ---- host tables (pinned: they are the H2D sources) ----
    Pin<int64_t> n_total, n_avail;             // [D][maxN]
    Pin<uint64_t> n_taint, n_label;
    Pin<uint32_t> n_flags;                     // bit0 schedulable, bit1 reserved (0 when absent)
    std::vector<uint32_t> n_rank;
    std::vector<uint8_t> n_present;
    uint32_t n_hi = 0;                         // 1 + highest node index in use
    bool nodes_stale = true, rank_stale = true;
    Pin<uint32_t> by_rank; uint32_t nlive = 0;
    bool ranks_unique = true;                // no two live nodes share a NodeID rank (checked where by_rank is rebuilt)

    Pin<int64_t> a_req;                        // [D][maxA]
    Pin<uint64_t> a_tol, a_need, a_deny;
    Pin<uint32_t> a_node;
    std::vector<int32_t> a_prio;
    std::vector<int64_t> a_create;
    std::vector<uint64_t> a_sig;    // signature hash of each ask's predicate inputs (yk::ask_signature)
    yk::RowShare share;
    bool share_rows = true;
    uint64_t split_min_pairs = 1ull << 25;   // multi-GPU: batches with fewer (row,node) pairs are swept whole on every rank
    std::vector<uint32_t> a_app, a_flags, a_gang, a_bound;
    std::vector<uint8_t> a_state;              // yk::ST_*, ST_ABSENT when not present
    uint32_t a_hi = 0;
    bool asks_stale = true;

    std::vector<uint32_t> p_queue; std::vector<int64_t> p_submit, p_alloc; std::vector<uint8_t> p_present;
    uint32_t nq = 0;
    std::vector<uint32_t> q_parent; std::vector<int64_t> q_guar, q_max, q_alloc; std::vector<uint8_t> q_sort;
    std::vector<int32_t> q_prio_offset; std::vector<uint8_t> q_prio_fence;   // queue properties priority.offset / priority.policy=fence
    std::vector<uint32_t> p_user, ul_queue, ul_user; std::vector<int64_t> ul_max, ul_alloc; uint32_t n_ul = 0;   // user / group limits

    // ---- device ----
    Dev<int64_t> d_total, d_avail; Dev<uint64_t> d_taint, d_label; Dev<uint32_t> d_flags, d_by_rank;
    Dev<int64_t> d_areq; Dev<uint64_t> d_atol, d_aneed, d_adeny; Dev<uint32_t> d_anode;
    Dev<uint64_t> d_key_in, d_key_out; Dev<uint32_t> d_val_in, d_val_out;
    Dev<uint8_t> d_cub; size_t cub_bytes = 0;
    Dev<int64_t> d_scap; Dev<uint64_t> d_staint, d_slabel; Dev<uint32_t> d_snode;
    Dev<int> d_flag;
    Slot slot[2];
    Worker worker;
    std::vector<uint32_t> pending;           // asks of the current cycle
    yk_stats_t wst{};                        // counters written by the worker thread, merged at join
    Dev<uint32_t> d_dirty_nodes; Dev<int64_t> d_dirty_vals; Dev<double> d_scores;
    size_t Wmax = 0;

    // pinned staging
    Pin<uint32_t> h_snode, h_dirty_nodes; Pin<uint64_t> h_skey; Pin<int64_t> h_dirty_vals;
    Pin<int> h_flag; Pin<double> h_scores;

    // ordered commit (host logic, csrc/yk_commit.hpp): working copy of the nodes, touched-node index, epoch state
    yk::Committer cm;
    Pin<uint32_t> h_order[2]; int cur = 0;   // node order (ascending (score, NodeID)), double-buffered
    Dev<uint32_t> d_order;
    int epochW = 0;                          // words per fit row in the current epoch
    uint32_t epoch_limit = 8192;             // an epoch ends before its touched-node count would pass this
    uint32_t epoch_floor = 8192, epoch_env = 0;
    bool prof = false;                       // YK_PROFILE_COMMIT: TSC split of the commit loop into st.dbg2[]
    bool no_spec = false;                    // debugging: never launch batch k+1 before batch k is committed
    int slots = 264;                         // resident sweep CTAs on this device (SMs x occupancy)

    yk::Orderer ord;
    // epoch rows: when the cycle's pending asks have few distinct predicate signatures, every signature is swept ONCE per
    // epoch (one launch, one read-back) and the batches of the epoch only index into those rows -- no per-batch device work
    static constexpr uint32_t EP_MAX = 1024;
    bool ep_rows = false; uint32_t ep_n = 0; bool ep_uploaded = false, ep_landed = true;
    std::vector<uint32_t> ep_reps;
    Dev<uint32_t> ep_d_batch, ep_d_fit; Pin<uint32_t> ep_h_batch, ep_h_fit;
    cudaEvent_t ep_ev = nullptr, ep_s0 = nullptr, ep_s1 = nullptr;
    SigTable sigs; std::vector<uint32_t> ep_local, ep_seen; uint32_t ep_stamp = 0;
    // device-resident ordered commit (yk_lattice.h): node records, ping-pong node order, per-batch staging
    bool lt_allowed = true;                  // !YK_FLAG_HOST_COMMIT, single GPU
    int lt_force = 0;                        // YK_FLAG_DEVICE_COMMIT / YK_COMMIT=device: every eligible cycle commits on the device
    bool lt_auto = false;                    // the default: eligible cycles whose order is made of long uniform runs commit on the device
    bool bp_device = false;                  // YK_FLAG_BINPACKING_DEVICE: binpacking cycles are eligible too (one fill per run)
    bool lt_active = false;                  // this cycle runs (so far) on the device commit
    bool cycle_has_gang = false;             // some pending ask of this cycle is a gang member
    bool order_enqueued = false;             // device_order() of this cycle is already on the stream
    int lt_RS = 0; size_t lt_smem = 0;
    Dev<int64_t> d_rec; Dev<yklt::Ent> d_ord[2]; Dev<int> d_lt_cur, d_lt_hdr; Dev<int64_t> d_lt_ub;
    Dev<uint32_t> d_rank, d_lt_asks, d_lt_meta, d_lt_shp, d_lt_sig, d_lt_res;
    Dev<long long> d_lt_prof; bool lt_prof = false; uint64_t lt_total_subruns = 0;   // YK_PROFILE_LATTICE: SM clocks per kernel phase, printed by yk_destroy
    Pin<uint32_t> h_lt_asks, h_lt_meta, h_lt_shp, h_lt_sig, h_lt_res; Pin<int> h_lt_hdr; Pin<int64_t> h_lt_ub;
    std::vector<uint32_t> a_shape, a_sigid;
    std::vector<uint8_t> a_cause;               // per ask: 0, ST_SLOWPATH or ST_INVALID (yk::Tables::a_cause), kept by yk_asks_upsert
    cudaEvent_t ev_l0 = nullptr, ev_l1 = nullptr;
    // uniform runs (yk_uniform.h): allocated on first use; element buffers hold UN_EMAX generated elements
    bool hp_on = false; double hp[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}; uint64_t hp_n = 0;
    bool un_alloc = false, un_ord_stale = false;   // un_ord_stale: uniform runs moved nodes since d_ord was last written
    int un_min = 2048;                          // shortest run that takes the uniform path (YK_UNIFORM_MIN)
    int un_depth = 0;                           // first depth of a uniform run's attempt (YK_UNIFORM_DEPTH); 0: ykun::first_depth
    Dev<unsigned long long> d_un_ekey[2], d_un_bk, d_un_rkey[2], d_un_rrn[2];
    Dev<uint32_t> d_un_enode[2], d_un_cnt;
    Dev<ykun::Globals> d_un_g; Pin<ykun::Globals> h_un_g;
    Dev<uint8_t> d_un_cub; size_t un_cub_bytes = 0;
    std::vector<ykun::Segment> un_segs;
    // round commit (yk_rounds.h) of mask-free stretches, automatic commit only
    int rd_min = yklt::RD_MIN;                  // fewest pending asks for which a mask-free cycle starts on it (YK_ROUND_MIN; 0: never)
    int rd_window = ykrd::WCAP;                 // candidates per round (YK_ROUND_WINDOW: a testing knob)
    int rd_guard = ykrd::GUARD;                  // asks per pass below which a stretch hands over to the host commit (YK_ROUND_GUARD)
    uint64_t rd_taints = 0;                     // this cycle: union of the live nodes' taints
    size_t rd_smem = 0;
    Dev<yklt::Ent> d_rd_spent; Dev<int> d_rd_hdr; Pin<int> h_rd_hdr;
    // mapped: the round kernel's results (indexed like the staged batch) and its decided count (ykrd::Args::prog), which the
    // host reads while the kernel runs
    Pin<uint32_t> h_rd_res; Pin<int> h_rd_prog;
    Dev<int64_t> d_rd_req;                      // [maxA][D]: a stretch's requests in stretch order (ykrd::Args::sreq)
    // speculative round-commit launch (yk_spec.h): device copies of what the static order needs (uploaded with the ask and
    // application tables when they are stale; the ask states every cycle), the order's own sort buffers and the screen's
    // words.  Mapped: the order and the words for the host's compare, and the abort word the kernel reads.
    bool sp_asks_stale = true, sp_apps_stale = true;
    bool sp_live = false;                       // a speculative launch of this cycle is on the stream
    bool sp_adopt = false;                      // ... and the host adopted it: lt_rounds takes it instead of launching
    std::vector<uint32_t> sp_pending;           // a speculative cycle's pending asks, listed on the calling thread
    Dev<uint32_t> d_sp_app, d_sp_gang, d_sp_sig; Dev<int64_t> d_sp_create, d_sp_submit; Dev<int32_t> d_sp_prio;
    Dev<uint8_t> d_sp_cause, d_sp_state, d_sp_present;
    Dev<uint64_t> d_sp_ckey[2], d_sp_pkey[2]; Dev<uint32_t> d_sp_cval[2], d_sp_ukey[2], d_sp_pval[2], d_sp_pos, d_sp_brk[2], d_sp_w;
    Dev<uint8_t> d_sp_cub; size_t sp_cub_bytes = 0;
    Pin<uint8_t> h_sp_state; Pin<uint32_t> h_sp_order, h_sp_w, h_sp_init; Pin<int> h_sp_abort;
    cudaEvent_t ev_sp = nullptr;                // after the screen: the order, the words and the NaN flag have landed
    Dev<uint32_t> pre_q; Dev<int64_t> pre_v; Dev<int32_t> pre_o;   // yk_preemption_search staging, grown on demand
    // yk_filter_nodes: its own node order (so a cycle's sort buffers are never touched) and per-chunk buffers, grown on demand
    Dev<uint64_t> f_key_in, f_key_out; Dev<uint32_t> f_val_in, f_val_out; Dev<uint8_t> f_cub; size_t f_cub_bytes = 0;
    Dev<int> f_flag; Pin<int> h_f_flag;
    Dev<uint32_t> f_asks, f_bits, f_tcnt, f_counts, f_out;
    Pin<uint32_t> h_f_asks, h_f_counts, h_f_out;
    // yk_preemption_nodes: node positions, per-chunk entry / group buffers and staging, grown on demand; pn_seen / pn_stamp find
    // a victim named twice in one list
    Dev<uint32_t> pn_pos, pn_in, pn_val_in, pn_val_out, pn_head, pn_incl, pn_gask, pn_gnode, pn_goff, pn_start, pn_out;
    Dev<uint64_t> pn_key_in, pn_key_out; Dev<int64_t> pn_vreq; Dev<int32_t> pn_res; Dev<uint8_t> pn_cub;
    Pin<uint32_t> h_pn_in, h_pn_out;
    std::vector<uint32_t> pn_seen; uint32_t pn_stamp = 0;
    // yk_preemption_plan: the queues' preemption fence, the marked victims and each planned preemptor's node (YK_NONE: none);
    // per-call device tables (queues, bound allocations, room), per-preemptor sort buffers and results, grown on demand
    std::vector<uint8_t> q_pp_fence, pp_mark; std::vector<uint32_t> pp_plan;
    Dev<uint32_t> pp_q32, pp_v32, pp_tv[2], pp_nkey[2], pp_nval[2], pp_seg, pp_cnt, pp_pnode; Dev<int32_t> pp_vprio;
    Dev<int64_t> pp_q64, pp_room, pp_pval; Dev<uint64_t> pp_key[2]; Dev<unsigned long long> pp_best;
    Dev<uint8_t> pp_hasg, pp_taken, pp_cub;
    // yk_preemption_required_node: per-call device tables (slots, groups, preemptors, sort buffers, results), grown on demand
    Dev<uint32_t> prn_u32, prn_val[2], prn_out; Dev<int32_t> prn_i32; Dev<int64_t> prn_room; Dev<uint64_t> prn_key[2];
    Dev<uint8_t> prn_taken, prn_cub;
    yk_allgather_fn xfn = nullptr; void* xctx = nullptr;
    // peer-to-peer exchange (see yk_peer_export): peers' slot buffers and sync blocks, mapped through CUDA IPC
    bool p2p = false;
    uint32_t seq = 0;
    Dev<uint32_t> d_sync;                    // [32]: ready[slot][rank] at slot*8+rank, consumed[slot][rank] at 16+slot*8+rank
    uint32_t* peer_fit[2][8] = {};
    uint32_t* peer_sync[8] = {};
    bool peer_open[8] = {};

    int fail(int code, const std::string& m) { err = m; return code; }
    int cuda_fail(cudaError_t e, const char* what) {
        err = std::string(what) + ": " + cudaGetErrorString(e);
        return YK_ERR_CUDA;
    }
};

#define CK(call)                                                     \
    do {                                                             \
        cudaError_t _e = (call);                                     \
        if (_e != cudaSuccess) return e->cuda_fail(_e, #call);       \
    } while (0)

namespace {

template <int D>
cudaError_t lattice_setup_d(size_t* smem) {
    *smem = sizeof(yklt::Shared<D>);
    return cudaFuncSetAttribute(yk_lattice_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem);
}
cudaError_t lattice_setup(int D, size_t* smem) {
    switch (D) {
        case 1: return lattice_setup_d<1>(smem); case 2: return lattice_setup_d<2>(smem); case 3: return lattice_setup_d<3>(smem);
        case 4: return lattice_setup_d<4>(smem); case 5: return lattice_setup_d<5>(smem); case 6: return lattice_setup_d<6>(smem);
        case 7: return lattice_setup_d<7>(smem); default: return lattice_setup_d<8>(smem);
    }
}
void launch_lattice(int D, const yklt::Args& a, size_t smem, cudaStream_t s) {
    switch (D) {
        case 1: yk_lattice_kernel<1><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 2: yk_lattice_kernel<2><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 3: yk_lattice_kernel<3><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 4: yk_lattice_kernel<4><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 5: yk_lattice_kernel<5><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 6: yk_lattice_kernel<6><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 7: yk_lattice_kernel<7><<<1, yklt::THREADS, smem, s>>>(a); break;
        default: yk_lattice_kernel<8><<<1, yklt::THREADS, smem, s>>>(a); break;
    }
}
template <int D>
cudaError_t rounds_setup_d(size_t smem) {
    return cudaFuncSetAttribute(yk_rounds_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}
cudaError_t rounds_setup(int D, size_t* smem) {
    *smem = sizeof(ykrd::Shared);
    switch (D) {
        case 1: return rounds_setup_d<1>(*smem); case 2: return rounds_setup_d<2>(*smem); case 3: return rounds_setup_d<3>(*smem);
        case 4: return rounds_setup_d<4>(*smem); case 5: return rounds_setup_d<5>(*smem); case 6: return rounds_setup_d<6>(*smem);
        case 7: return rounds_setup_d<7>(*smem); default: return rounds_setup_d<8>(*smem);
    }
}
void launch_rounds(int D, const ykrd::Args& a, size_t smem, cudaStream_t s) {
    switch (D) {
        case 1: yk_rounds_kernel<1><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 2: yk_rounds_kernel<2><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 3: yk_rounds_kernel<3><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 4: yk_rounds_kernel<4><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 5: yk_rounds_kernel<5><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 6: yk_rounds_kernel<6><<<1, yklt::THREADS, smem, s>>>(a); break;
        case 7: yk_rounds_kernel<7><<<1, yklt::THREADS, smem, s>>>(a); break;
        default: yk_rounds_kernel<8><<<1, yklt::THREADS, smem, s>>>(a); break;
    }
}

int upload_tables(yk_engine* e) {
    const int D = e->D;
    if (e->rank_stale) {
        std::vector<uint32_t> live;
        live.reserve(e->n_hi);
        for (uint32_t i = 0; i < e->n_hi; ++i) if (e->n_present[i]) live.push_back(i);
        std::sort(live.begin(), live.end(), [&](uint32_t a, uint32_t b) {
            if (e->n_rank[a] != e->n_rank[b]) return e->n_rank[a] < e->n_rank[b];
            return a < b;
        });
        e->nlive = (uint32_t)live.size();
        e->ranks_unique = true;
        for (size_t i = 1; i < live.size(); ++i) if (e->n_rank[live[i]] == e->n_rank[live[i - 1]]) e->ranks_unique = false;
        if (e->nlive) memcpy(e->by_rank.p, live.data(), sizeof(uint32_t) * e->nlive);
        if (e->nlive) CK(cudaMemcpyAsync(e->d_by_rank.p, e->by_rank.p, sizeof(uint32_t) * e->nlive, cudaMemcpyHostToDevice, e->stream));
        e->st.h2d_bytes += sizeof(uint32_t) * e->nlive;
        if (e->lt_allowed && e->n_hi) {   // the lattice commit orders ties by the rank itself
            CK(cudaMemcpyAsync(e->d_rank.p, e->n_rank.data(), sizeof(uint32_t) * e->n_hi, cudaMemcpyHostToDevice, e->stream));
            CK(cudaStreamSynchronize(e->stream));   // n_rank is pageable memory
            e->st.h2d_bytes += sizeof(uint32_t) * e->n_hi;
        }
        e->rank_stale = false;
    }
    if (e->nodes_stale && e->n_hi) {
        const size_t n = e->n_hi;
        for (int k = 0; k < D; ++k) {
            CK(cudaMemcpyAsync(e->d_total.p + (size_t)k * e->maxN, e->n_total.p + (size_t)k * e->maxN, 8 * n, cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemcpyAsync(e->d_avail.p + (size_t)k * e->maxN, e->n_avail.p + (size_t)k * e->maxN, 8 * n, cudaMemcpyHostToDevice, e->stream));
        }
        CK(cudaMemcpyAsync(e->d_taint.p, e->n_taint.p, 8 * n, cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->d_label.p, e->n_label.p, 8 * n, cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->d_flags.p, e->n_flags.p, 4 * n, cudaMemcpyHostToDevice, e->stream));
        e->st.h2d_bytes += n * (16 * D + 20);
    }
    e->nodes_stale = false;
    if (e->asks_stale && e->a_hi) {
        const size_t n = e->a_hi;
        for (int k = 0; k < D; ++k)
            CK(cudaMemcpyAsync(e->d_areq.p + (size_t)k * e->maxA, e->a_req.p + (size_t)k * e->maxA, 8 * n, cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->d_atol.p, e->a_tol.p, 8 * n, cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->d_aneed.p, e->a_need.p, 8 * n, cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->d_adeny.p, e->a_deny.p, 8 * n, cudaMemcpyHostToDevice, e->stream));
        CK(cudaMemcpyAsync(e->d_anode.p, e->a_node.p, 4 * n, cudaMemcpyHostToDevice, e->stream));
        e->st.h2d_bytes += n * (8 * D + 28);
        e->sp_asks_stale = true;
    }
    e->asks_stale = false;
    // the speculative order's tables, where a cycle may start on the round commit (spec_gate)
    if (e->lt_allowed && e->lt_auto && !e->lt_force && e->rd_min > 0 && e->un_min > 0) {
        if (e->sp_asks_stale && e->a_hi) {
            const size_t n = e->a_hi;
            CK(cudaMemcpyAsync(e->d_sp_app.p, e->a_app.data(), 4 * n, cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemcpyAsync(e->d_sp_create.p, e->a_create.data(), 8 * n, cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemcpyAsync(e->d_sp_prio.p, e->a_prio.data(), 4 * n, cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemcpyAsync(e->d_sp_gang.p, e->a_gang.data(), 4 * n, cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemcpyAsync(e->d_sp_cause.p, e->a_cause.data(), n, cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemcpyAsync(e->d_sp_sig.p, e->a_sigid.data(), 4 * n, cudaMemcpyHostToDevice, e->stream));
            e->st.h2d_bytes += n * 25;
        }
        if (e->sp_apps_stale) {
            CK(cudaMemcpyAsync(e->d_sp_submit.p, e->p_submit.data(), 8 * (size_t)e->maxP, cudaMemcpyHostToDevice, e->stream));
            CK(cudaMemcpyAsync(e->d_sp_present.p, e->p_present.data(), e->maxP, cudaMemcpyHostToDevice, e->stream));
            e->st.h2d_bytes += 9 * (size_t)e->maxP;
        }
        if (e->sp_asks_stale || e->sp_apps_stale) CK(cudaStreamSynchronize(e->stream));   // the sources are pageable
        e->sp_asks_stale = e->sp_apps_stale = false;
    }
    return YK_OK;
}

// grid.y (ask splits) is sized so that tiles x splits fills the resident CTA slots of the device exactly once
template <int D>
void launch_sweep_d(YkSweepArgs a, cudaStream_t s, int slots) {
    const int tiles = a.Np / NODE_TILE;
    int splits = std::max(1, slots / tiles);
    a.per = (a.rows + splits - 1) / splits;
    splits = (a.rows + a.per - 1) / a.per;
    dim3 grid((unsigned)tiles, (unsigned)splits);
    yk_sweep_kernel<D, NPT, AC><<<grid, YK_SWEEP_THREADS, 0, s>>>(a);
}
template <int D>
int sweep_slots_d(int sms) {
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, yk_sweep_kernel<D, NPT, AC>, YK_SWEEP_THREADS, 0) != cudaSuccess || per_sm < 1) per_sm = 2;
    return per_sm * sms;
}
int sweep_slots(int D, int sms) {
    switch (D) {
        case 1: return sweep_slots_d<1>(sms); case 2: return sweep_slots_d<2>(sms); case 3: return sweep_slots_d<3>(sms);
        case 4: return sweep_slots_d<4>(sms); case 5: return sweep_slots_d<5>(sms); case 6: return sweep_slots_d<6>(sms);
        case 7: return sweep_slots_d<7>(sms); default: return sweep_slots_d<8>(sms);
    }
}
void launch_sweep(int D, const YkSweepArgs& a, cudaStream_t s, int slots) {
    switch (D) {
        case 1: launch_sweep_d<1>(a, s, slots); break;
        case 2: launch_sweep_d<2>(a, s, slots); break;
        case 3: launch_sweep_d<3>(a, s, slots); break;
        case 4: launch_sweep_d<4>(a, s, slots); break;
        case 5: launch_sweep_d<5>(a, s, slots); break;
        case 6: launch_sweep_d<6>(a, s, slots); break;
        case 7: launch_sweep_d<7>(a, s, slots); break;
        default: launch_sweep_d<8>(a, s, slots); break;
    }
}

// Initial node order of a cycle, computed on the device: float64 score per node (yk_key_kernel), stable radix
// sort by key over NodeID-rank order = ascending (score, NodeID).  device_order() only enqueues (the lattice commit
// consumes the result on the stream); initial_order() also brings it to the host commit's working copy.
void setup_commit_tables(yk_engine* e) {
    yk::CommitTables& ct = e->cm.t;
    ct.D = e->D; ct.policy = e->cfg.policy; ct.w = e->w.w; ct.lda = e->maxA;
    ct.a_req = e->a_req.p; ct.a_tol = e->a_tol.p; ct.a_need = e->a_need.p; ct.a_deny = e->a_deny.p; ct.a_node = e->a_node.p;
    ct.a_gang = e->a_gang.data(); ct.a_app = e->a_app.data();
    e->cm.profile = e->prof;
}

int device_order(yk_engine* e) {
    const int nlive = (int)e->nlive;
    if (nlive == 0) return YK_OK;
    cudaStream_t s = e->stream;
    CK(cudaMemsetAsync(e->d_flag.p, 0, sizeof(int), s));
    CK(cudaEventRecord(e->ev0, s));
    yk_key_kernel<<<(nlive + 255) / 256, 256, 0, s>>>(e->D, e->cfg.policy, e->w, e->d_total.p, e->d_avail.p, e->maxN,
                                                     e->d_by_rank.p, nlive, e->d_key_in.p, e->d_val_in.p, e->d_flag.p);
    size_t tb = e->cub_bytes;
    CK(cub::DeviceRadixSort::SortPairs(e->d_cub.p, tb, e->d_key_in.p, e->d_key_out.p, e->d_val_in.p, e->d_val_out.p,
                                       nlive, 0, 64, s));
    CK(cudaEventRecord(e->ev1, s));
    CK(cudaMemcpyAsync(e->h_flag.p, e->d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    e->st.d2h_bytes += 4;
    e->st.other_launches += 11;   // key + cub radix sort (histogram, exclusive sum, 8 onesweep passes for 64-bit keys)
    return YK_OK;
}

int initial_order(yk_engine* e) {
    const int nlive = (int)e->nlive;
    if (nlive == 0) return YK_OK;
    cudaStream_t s = e->stream;
    if (!e->order_enqueued) {   // (after a hand-over from the device commit the order is computed again from the exported tables)
        int rc = device_order(e);
        if (rc) return rc;
    }
    e->order_enqueued = false;
    CK(cudaMemcpyAsync(e->h_order[0].p, e->d_val_out.p, sizeof(uint32_t) * (size_t)nlive, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(e->h_skey.p, e->d_key_out.p, sizeof(uint64_t) * (size_t)nlive, cudaMemcpyDeviceToHost, s));
    // while the device scores and sorts: the commit's working copy of the node table (host only)
    e->cm.build(e->n_hi, e->n_avail.p, e->n_total.p, e->maxN, e->n_taint.p, e->n_label.p, e->n_rank.data());
    CK(cudaStreamSynchronize(s));
    e->st.d2h_bytes += 12 * (size_t)nlive;
    if (e->h_flag[0]) return e->fail(YK_ERR_RANGE, "NaN node score (zero total on a weighted resource)");
    float ms = 0;
    cudaEventElapsedTime(&ms, e->ev0, e->ev1);
    e->st.sort_ms += ms;
    e->cur = 0;
    e->cm.set_order(e->h_order[0].p, e->h_skey.p, nlive);   // the cycle's initial order: (key, rank, node) per position
    return YK_OK;
}

// ---- uniform runs on the device (yk_uniform.h / yk_uniform.cuh) -------------------------------------------------------
int un_ensure(yk_engine* e) {
    if (e->un_alloc) return YK_OK;
    const size_t N = e->maxN;
    for (int b = 0; b < 2; ++b) {
        CK(e->d_un_ekey[b].alloc(ykun::UN_EMAX)); CK(e->d_un_enode[b].alloc(ykun::UN_EMAX));
        CK(e->d_un_rkey[b].alloc(N)); CK(e->d_un_rrn[b].alloc(N));
    }
    CK(e->d_un_bk.alloc(N)); CK(e->d_un_cnt.alloc(N));
    CK(e->d_un_g.alloc(1)); CK(e->h_un_g.alloc(1));
    CK(cudaMemsetAsync(e->d_un_cnt.p, 0, sizeof(uint32_t) * std::max<size_t>(N, 1), e->stream));
    size_t t0 = 0, t1 = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, t0, e->d_un_ekey[0].p, e->d_un_ekey[1].p, e->d_un_enode[0].p, e->d_un_enode[1].p, (int)ykun::UN_EMAX, 0, 64, e->stream));
    CK(cub::DeviceRadixSort::SortPairs(nullptr, t1, e->d_un_rkey[0].p, e->d_un_rkey[1].p, e->d_un_rrn[0].p, e->d_un_rrn[1].p, (int)std::max<size_t>(N, 1), 0, 64, e->stream));
    size_t t2 = 0;   // the binpacking fill's scan
    CK(cub::DeviceScan::InclusiveSum(nullptr, t2, e->d_un_rkey[0].p, e->d_un_rkey[1].p, (int)std::max<size_t>(N, 1), e->stream));
    e->un_cub_bytes = std::max(std::max(t0, t1), t2);
    CK(e->d_un_cub.alloc(e->un_cub_bytes));
    e->un_alloc = true;
    return YK_OK;
}

template <int D>
cudaError_t un_attempt_d(yk_engine* e, const ykun::Args& a) {
    cudaStream_t s = e->stream;
    const int nb = (a.nlive + 255) / 256;
    ykun::un_reset_kernel<<<1, 1, 0, s>>>(a.g);
    ykun::un_depth_kernel<D><<<(unsigned)(((size_t)a.nlive * (size_t)a.L + 255) / 256), 256, 0, s>>>(a);
    ykun::un_brank_kernel<D><<<nb, 256, 0, s>>>(a);
    size_t tb = e->un_cub_bytes;
    cudaError_t rc = cub::DeviceRadixSort::SortPairs(e->d_un_cub.p, tb, a.ekey, const_cast<unsigned long long*>(a.skey), a.enode,
                                                     const_cast<uint32_t*>(a.snode), a.nlive * a.L, 0, 64, s);
    if (rc != cudaSuccess) return rc;
    ykun::un_select_kernel<D><<<(a.R + 255) / 256, 256, 0, s>>>(a);
    ykun::un_decide_kernel<<<1, 1, 0, s>>>(a);
    ykun::un_apply_rekey_kernel<D><<<nb, 256, 0, s>>>(a);   // leaves the new order entries (rank order) in rkey / rrn
    return cudaGetLastError();
}
cudaError_t un_attempt(yk_engine* e, const ykun::Args& a) {
    switch (e->D) {
        case 1: return un_attempt_d<1>(e, a); case 2: return un_attempt_d<2>(e, a); case 3: return un_attempt_d<3>(e, a);
        case 4: return un_attempt_d<4>(e, a); case 5: return un_attempt_d<5>(e, a); case 6: return un_attempt_d<6>(e, a);
        case 7: return un_attempt_d<7>(e, a); default: return un_attempt_d<8>(e, a);
    }
}

// One binpacking fill (yk_uniform.h): the run's keys at L = 1, sorted; capacities per sorted position, scanned; decide,
// select, apply.  Once the keys are sorted, ekey holds the capacities and bk their inclusive sum.
template <int D>
cudaError_t un_fill_d(yk_engine* e, const ykun::Args& a) {
    cudaStream_t s = e->stream;
    const int nb = (a.nlive + 255) / 256;
    ykun::un_reset_kernel<<<1, 1, 0, s>>>(a.g);
    ykun::un_depth_kernel<D><<<nb, 256, 0, s>>>(a);   // a.L == 1
    size_t tb = e->un_cub_bytes;
    cudaError_t rc = cub::DeviceRadixSort::SortPairs(e->d_un_cub.p, tb, a.ekey, const_cast<unsigned long long*>(a.skey), a.enode,
                                                     const_cast<uint32_t*>(a.snode), a.nlive, 0, 64, s);
    if (rc != cudaSuccess) return rc;
    ykun::un_fill_cap_kernel<D><<<nb, 256, 0, s>>>(a);
    tb = e->un_cub_bytes;
    rc = cub::DeviceScan::InclusiveSum(e->d_un_cub.p, tb, a.ekey, a.bk, a.nlive, s);
    if (rc != cudaSuccess) return rc;
    ykun::un_fill_decide_kernel<<<1, 1, 0, s>>>(a);
    ykun::un_fill_select_kernel<<<(a.R + 255) / 256, 256, 0, s>>>(a);
    ykun::un_apply_rekey_kernel<D><<<nb, 256, 0, s>>>(a);
    return cudaGetLastError();
}
cudaError_t un_fill(yk_engine* e, const ykun::Args& a) {
    switch (e->D) {
        case 1: return un_fill_d<1>(e, a); case 2: return un_fill_d<2>(e, a); case 3: return un_fill_d<3>(e, a);
        case 4: return un_fill_d<4>(e, a); case 5: return un_fill_d<5>(e, a); case 6: return un_fill_d<6>(e, a);
        case 7: return un_fill_d<7>(e, a); default: return un_fill_d<8>(e, a);
    }
}

// The node order after uniform runs: only the windowed kernel reads it, so it is rebuilt (stable sort of the re-keyed entries,
// which un_apply_rekey_kernel left in rank order) when a windowed stretch follows, not after every run.
int un_reorder(yk_engine* e) {
    if (!e->un_ord_stale) return YK_OK;
    cudaStream_t s = e->stream;
    const int nlive = (int)e->nlive;
    size_t tb = e->un_cub_bytes;
    CK(cub::DeviceRadixSort::SortPairs(e->d_un_cub.p, tb, e->d_un_rkey[0].p, e->d_un_rkey[1].p, e->d_un_rrn[0].p, e->d_un_rrn[1].p, nlive, 0, 64, s));
    ykun::Args a{};
    a.ord[0] = e->d_ord[0].p; a.ord[1] = e->d_ord[1].p; a.cur = e->d_lt_cur.p; a.nlive = nlive;
    a.okey = e->d_un_rkey[1].p; a.orn = e->d_un_rrn[1].p;
    ykun::un_order_kernel<<<(nlive + 255) / 256, 256, 0, s>>>(a);
    CK(cudaGetLastError());
    e->st.other_launches += 11;
    e->un_ord_stale = false;
    return YK_OK;
}

// One uniform run: entries [off, off + R) of the staged batch (h_lt_asks; results land in d_lt_res at the same offset),
// through ykun::uniform_run with un_attempt as the attempt (un_fill under binpacking).
int lt_uniform(yk_engine* e, size_t off, size_t R, bool has_gang, int* status, size_t* consumed) {
    const int nlive = (int)e->nlive;
    int rc = un_ensure(e);
    if (rc) return rc;
    cudaStream_t s = e->stream;
    const uint32_t ask = e->h_lt_asks[off];
    ykun::Args a{};
    a.policy = e->cfg.policy;
    for (int k = 0; k < 8; ++k) { a.w[k] = e->w.w[k]; a.req[k] = k < e->D ? e->a_req[(size_t)k * e->maxA + ask] : 0; }
    a.rec = e->d_rec.p; a.RS = e->lt_RS; a.ord[0] = e->d_ord[0].p; a.ord[1] = e->d_ord[1].p; a.cur = e->d_lt_cur.p;
    a.nlive = nlive; a.byrank = e->d_by_rank.p;   // live nodes by ascending (NodeID rank, index): upload_tables
    a.tol = e->a_tol[ask]; a.need = e->a_need[ask]; a.deny = e->a_deny[ask]; a.want = e->a_node[ask];
    a.R = (int)R; a.insensitive = e->ord.insensitive ? 1 : 0; a.has_gang = has_gang ? 1 : 0;
    a.ekey = e->d_un_ekey[0].p; a.skey = e->d_un_ekey[1].p; a.enode = e->d_un_enode[0].p; a.snode = e->d_un_enode[1].p;
    a.bk = e->d_un_bk.p; a.cnt = e->d_un_cnt.p;
    a.rkey = e->d_un_rkey[0].p; a.okey = e->d_un_rkey[1].p; a.rrn = e->d_un_rrn[0].p; a.orn = e->d_un_rrn[1].p;
    a.res = e->d_lt_res.p + off; a.g = e->d_un_g.p;
    const bool bp = e->cfg.policy == YK_POLICY_BINPACKING;
    auto attempt = [&](int L, ykun::Globals& g) -> int {
        a.L = L;
        CK(cudaEventRecord(e->ev_l0, s));
        CK(bp ? un_fill(e, a) : un_attempt(e, a));
        CK(cudaEventRecord(e->ev_l1, s));
        CK(cudaMemcpyAsync(e->h_un_g.p, e->d_un_g.p, sizeof(ykun::Globals), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        float ms = 0;
        cudaEventElapsedTime(&ms, e->ev_l0, e->ev_l1);
        e->st.lattice_ms += ms;
        e->st.lattice_launches += 1;
        // 6 kernels of yk_uniform.cuh + one cub radix sort (histogram, exclusive sum, 8 onesweep passes); a fill: 6 kernels, the
        // sort, a cub scan (init, scan)
        e->st.other_launches += bp ? 18 : 16;
        e->st.d2h_bytes += sizeof(ykun::Globals);
        g = e->h_un_g[0];
        return YK_OK;
    };
    rc = ykun::uniform_run(e->D, e->w.w, a.req, e->n_total.p, e->maxN, e->by_rank.p, nlive, (int)R, e->un_depth, e->st, attempt,
                           status, consumed, bp);
    if (*status == ykun::U_DONE || *status == ykun::U_STOPPED) e->un_ord_stale = true;
    return rc;
}

// ---- device-resident ordered commit (yk_lattice.h) -------------------------------------------------------------------
// node records + order entries from the sorted keys; capacity bound and header reset
int lt_prepare(yk_engine* e) {
    const int nlive = (int)e->nlive;
    cudaStream_t s = e->stream;
    if (nlive)
        yk_lt_init_kernel<<<(nlive + 255) / 256, 256, 0, s>>>(e->D, e->d_total.p, e->d_avail.p, e->maxN, e->d_taint.p, e->d_label.p,
                                                             e->d_flags.p, e->d_rank.p, e->d_key_out.p, e->d_val_out.p, nlive,
                                                             e->d_rec.p, e->lt_RS, e->d_ord[0].p);
    CK(cudaGetLastError());
    for (int k = 0; k < 8; ++k) e->h_lt_ub[(size_t)k] = INT64_MAX;
    CK(cudaMemcpyAsync(e->d_lt_ub.p, e->h_lt_ub.p, 8 * sizeof(int64_t), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(e->d_lt_cur.p, 0, sizeof(int), s));
    CK(cudaMemsetAsync(e->d_lt_hdr.p, 0, yklt::H_WORDS * sizeof(int), s));
    e->st.other_launches += 1;
    memset(e->h_lt_hdr.p, 0, yklt::H_WORDS * sizeof(int));
    e->un_ord_stale = false;
    return YK_OK;
}

// One stretch [off, off + B) of the staged batch through yk_lattice_kernel; its header comes back into h_lt_hdr.
int lt_window(yk_engine* e, size_t off, size_t B) {
    cudaStream_t s = e->stream;
    { const int rco = un_reorder(e); if (rco) return rco; }
    yklt::Args a{};
    a.policy = e->cfg.policy;
    for (int k = 0; k < 8; ++k) a.w[k] = e->w.w[k];
    a.rec = e->d_rec.p; a.RS = e->lt_RS; a.ord[0] = e->d_ord[0].p; a.ord[1] = e->d_ord[1].p; a.cur = e->d_lt_cur.p;
    a.nlive = (int)e->nlive;
    a.a_req = e->d_areq.p; a.lda = e->maxA; a.a_tol = e->d_atol.p; a.a_need = e->d_aneed.p; a.a_deny = e->d_adeny.p; a.a_node = e->d_anode.p;
    a.asks = e->d_lt_asks.p + off; a.meta = e->d_lt_meta.p + off; a.shp = e->d_lt_shp.p + off; a.sig = e->d_lt_sig.p + off; a.B = (int)B;
    a.res = e->d_lt_res.p + off; a.hdr = e->d_lt_hdr.p; a.ub = e->d_lt_ub.p; a.insensitive = e->ord.insensitive ? 1 : 0;
    a.prof = e->lt_prof ? e->d_lt_prof.p : nullptr;
    CK(cudaEventRecord(e->ev_l0, s));
    launch_lattice(e->D, a, e->lt_smem, s);
    CK(cudaGetLastError());
    CK(cudaEventRecord(e->ev_l1, s));
    CK(cudaMemcpyAsync(e->h_lt_hdr.p, e->d_lt_hdr.p, yklt::H_WORDS * sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    float ms = 0;
    cudaEventElapsedTime(&ms, e->ev_l0, e->ev_l1);
    e->st.lattice_ms += ms;
    e->st.lattice_launches += 1;
    e->st.d2h_bytes += yklt::H_WORDS * sizeof(int);
    return YK_OK;
}

// One round-eligible stretch [off, off + B) of the staged batch through yk_rounds_kernel.  Its results land in the mapped
// h_rd_res at the same offset; while the kernel runs, ahead(off, to) is called for every newly published decided prefix
// [off, to), which the caller settles behind the kernel (yklt::settle_ahead).
// The round kernel over the staged stretch [off, off + B) (a.go etc. null), with its events and the header's read-back
int launch_stretch(yk_engine* e, size_t off, size_t B, const ykrd::Args* spec = nullptr) {
    cudaStream_t s = e->stream;
    ykrd::Args a{};
    if (spec) a = *spec;
    a.policy = e->cfg.policy;
    for (int k = 0; k < 8; ++k) a.w[k] = e->w.w[k];
    a.rec = e->d_rec.p; a.RS = e->lt_RS; a.ord[0] = e->d_ord[0].p; a.ord[1] = e->d_ord[1].p; a.cur = e->d_lt_cur.p;
    a.nlive = (int)e->nlive; a.spent = e->d_rd_spent.p;
    a.a_req = e->d_areq.p; a.lda = e->maxA; a.a_tol = e->d_atol.p; a.a_need = e->d_aneed.p; a.a_deny = e->d_adeny.p; a.a_node = e->d_anode.p;
    a.asks = e->d_lt_asks.p + off; a.B = (int)B; a.sreq = e->d_rd_req.p; a.res = e->h_rd_res.d + off; a.hdr = e->d_rd_hdr.p;
    a.prog = e->h_rd_prog.d;
    a.window = std::max(1, std::min(e->rd_window, ykrd::WCAP)); a.guard = e->rd_guard;
    a.prof = e->lt_prof ? e->d_lt_prof.p + 16 : nullptr;
    __atomic_store_n(e->h_rd_prog.p, 0, __ATOMIC_RELAXED);   // (no kernel that writes it is in flight)
    CK(cudaEventRecord(e->ev_l0, s));
    launch_rounds(e->D, a, e->rd_smem, s);
    CK(cudaGetLastError());
    CK(cudaEventRecord(e->ev_l1, s));
    CK(cudaMemcpyAsync(e->h_rd_hdr.p, e->d_rd_hdr.p, ykrd::R_WORDS * sizeof(int), cudaMemcpyDeviceToHost, s));
    return YK_OK;
}

template <class Ahead>
int lt_rounds(yk_engine* e, size_t off, size_t B, int* status, size_t* consumed, Ahead&& ahead) {
    cudaStream_t s = e->stream;
    { const int rco = un_reorder(e); if (rco) return rco; }
    // an adopted speculative launch (spec_verify) is this stretch, the batch's only one, already running
    const bool adopted = e->sp_adopt && off == 0;
    e->sp_adopt = false;
    if (!adopted) { const int rcl = launch_stretch(e, off, B); if (rcl) return rcl; }
    // settle behind the kernel until it ends; the count is read after the query, so the last pass sees its final value.  The
    // kernel never waits for the host: this loop only reads.
    for (size_t seen = 0;;) {
        const bool ended = cudaEventQuery(e->ev_l1) != cudaErrorNotReady;
        const size_t t = (size_t)__atomic_load_n(e->h_rd_prog.p, __ATOMIC_ACQUIRE);
        if (t > seen && t <= B) {
            const double t0 = e->hp_on ? now_ms() : 0;
            ahead(off, off + t);
            seen = t;
            if (e->hp_on) e->hp[7] += now_ms() - t0;   // YK_PROFILE_HOST: settle time hidden behind the kernel
        }
        if (ended) break;
    }
    CK(cudaStreamSynchronize(s));
    float ms = 0;
    cudaEventElapsedTime(&ms, e->ev_l0, e->ev_l1);
    e->st.lattice_ms += ms;
    e->st.lattice_launches += 1;
    e->st.d2h_bytes += ykrd::R_WORDS * sizeof(int);
    const int* h = e->h_rd_hdr.p;
    *status = h[ykrd::R_STATUS];
    *consumed = (size_t)h[ykrd::R_CONSUMED];
    if (*consumed > B) return e->fail(YK_ERR_CUDA, "round kernel returned a bad header");
    e->st.d2h_bytes += 4 * *consumed;   // the results, written straight into host memory
    e->st.round_passes += (uint64_t)h[ykrd::R_PASSES]; e->st.round_single_steps += (uint64_t)h[ykrd::R_SINGLES];
    e->st.round_asks += *consumed;
    return YK_OK;
}

// One batch of slot[0] (segments planned in e->un_segs) through yklt::run_segments; the decided entries' nodes land in
// `result`.  Blocks until it is decided; ahead(res, off, to) settles entries of a round stretch while its kernel runs (res:
// the batch's results as the round kernel writes them).
template <class Ahead>
int lt_batch(yk_engine* e, size_t B, int* status, size_t* done, std::vector<uint32_t>& result, Ahead&& ahead) {
    cudaStream_t s = e->stream;
    memcpy(e->h_lt_asks.p, e->slot[0].asks.data(), 4 * B);
    bool staged = false, asks_staged = e->sp_adopt;   // only the windowed kernel reads the per-entry words, the round kernel the
                                                       // asks (an adopted speculative launch wrote them itself)
    bool on_device = false;                     // some results are in d_lt_res (a uniform run or a windowed stretch)
    std::vector<std::pair<size_t, size_t>> in_host;   // the round stretches' [off, off + consumed): results in h_rd_res
    auto uniform = [&](size_t off, size_t len, bool has_gang, int* ust, size_t* consumed) {
        on_device = true;
        return lt_uniform(e, off, len, has_gang, ust, consumed);
    };
    auto window = [&](size_t off, size_t len, int* st, size_t* consumed) -> int {
        on_device = true;
        if (!staged) {
            CK(cudaMemcpyAsync(e->d_lt_asks.p, e->h_lt_asks.p, 4 * B, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(e->d_lt_meta.p, e->h_lt_meta.p, 4 * B, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(e->d_lt_shp.p, e->h_lt_shp.p, 4 * B, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(e->d_lt_sig.p, e->h_lt_sig.p, 4 * B, cudaMemcpyHostToDevice, s));
            e->st.h2d_bytes += 16 * B;
            staged = asks_staged = true;
        }
        const int rc = lt_window(e, off, len);
        if (rc) return rc;
        *st = e->h_lt_hdr[yklt::H_STATUS];
        *consumed = (size_t)e->h_lt_hdr[yklt::H_CONSUMED];
        if (*consumed > len) return e->fail(YK_ERR_CUDA, "lattice kernel returned a bad header");
        return YK_OK;
    };
    // the round commit takes the mask-free stretches of an automatic cycle; it reads the asks only
    auto rounds = [&](size_t off, size_t len, int* st, size_t* consumed) -> int {
        if (!asks_staged) {
            CK(cudaMemcpyAsync(e->d_lt_asks.p, e->h_lt_asks.p, 4 * B, cudaMemcpyHostToDevice, s));
            e->st.h2d_bytes += 4 * B;
            asks_staged = true;
        }
        const int rc = lt_rounds(e, off, len, st, consumed, [&](size_t o, size_t to) { ahead(e->h_rd_res.p, o, to); });
        if (!rc) in_host.emplace_back(off, *consumed);
        return rc;
    };
    const int rc = yklt::route_batch(e->cfg.policy == YK_POLICY_BINPACKING, !e->lt_force, e->cm.t, e->ord.insensitive, e->rd_taints,
                                     e->h_lt_asks.p, e->un_segs, e->h_lt_meta.p, uniform, rounds, window, status, done);
    if (rc) return rc;
    if (*done && on_device) {
        CK(cudaMemcpyAsync(e->h_lt_res.p, e->d_lt_res.p, 4 * *done, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        e->st.d2h_bytes += 4 * *done;
    }
    result.assign(e->h_lt_res.p, e->h_lt_res.p + B);
    for (const auto& r : in_host) std::copy(e->h_rd_res.p + r.first, e->h_rd_res.p + r.first + r.second, result.begin() + r.first);
    return YK_OK;
}

// the records' availability back into the column-major device table and the host table (end of the cycle, or hand-over)
int lt_export(yk_engine* e) {
    const int nlive = (int)e->nlive;
    if (nlive == 0) return YK_OK;
    cudaStream_t s = e->stream;
    yk_lt_export_kernel<<<(nlive + 255) / 256, 256, 0, s>>>(e->D, e->d_rec.p, e->lt_RS, e->d_ord[0].p, e->d_ord[1].p, e->d_lt_cur.p,
                                                            nlive, e->d_avail.p, e->maxN);
    CK(cudaGetLastError());
    for (int k = 0; k < e->D; ++k)
        CK(cudaMemcpyAsync(e->n_avail.p + (size_t)k * e->maxN, e->d_avail.p + (size_t)k * e->maxN, 8 * (size_t)e->n_hi, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    e->st.d2h_bytes += 8 * (size_t)e->n_hi * e->D;
    e->st.other_launches += 1;
    return YK_OK;
}

// ---- speculative round-commit launch (yk_spec.h, DESIGN.md §6.3) ----------------------------------------------------
// Cheap host gates, O(applications + queues), before the pending scan: a cycle under `auto` on the fair sort whose order can
// be placement-insensitive -- every present application in one fifo leaf with no max on its chain, no user limit, no queue
// priority offset or fence -- and with enough asks for the round commit.
bool spec_gate(const yk_engine* e, uint32_t max_bindings, bool auto_lattice) {
    if (!auto_lattice || e->cfg.policy != YK_POLICY_FAIR || e->rd_min <= 0 || max_bindings == 0 || e->a_hi < (uint32_t)e->rd_min || e->n_ul)
        return false;
    uint32_t leaf = YK_NONE;
    for (uint32_t p = 0; p < e->maxP; ++p) {
        if (!e->p_present[p]) continue;
        if (leaf == YK_NONE) leaf = e->p_queue[p];
        else if (e->p_queue[p] != leaf) return false;
    }
    if (leaf == YK_NONE || e->q_sort[leaf] != 0) return false;
    for (uint32_t q = 0; q < e->nq; ++q)
        if ((q > 0 && e->q_parent[q] == leaf) || e->q_prio_offset[q] != 0 || e->q_prio_fence[q]) return false;
    for (uint32_t q = leaf; q != YK_NONE; q = e->q_parent[q])
        for (int k = 0; k < e->D; ++k) if (e->q_max[(size_t)k * e->nq + q] != yk::UNSET) return false;
    return true;
}

// Enqueues, behind device_order: the static order of the kept asks into d_lt_asks (and h_sp_order), the screen, lt_prepare's
// set-up and the round kernel over the order, which returns at once unless the screen said GO and no node scores NaN.
// h_sp_state holds the ask states as the cycle began.  Needs the tables uploaded and the node order enqueued.
int spec_launch(yk_engine* e, uint32_t max_bindings) {
    if (!e->nlive || !e->ranks_unique) return YK_OK;
    for (int k = 0; k < e->D; ++k) if (!(e->w.w[k] >= 0.0)) return YK_OK;
    cudaStream_t s = e->stream;
    const uint32_t A = e->a_hi, P = e->maxP, n = std::max(std::max(A, e->nlive), P);
    CK(cudaMemcpyAsync(e->d_sp_state.p, e->h_sp_state.p, A, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(e->d_sp_w.p, e->h_sp_init.p, 4 * ykspec::W_N, cudaMemcpyHostToDevice, s));
    e->st.h2d_bytes += A + 4 * ykspec::W_N;
    yk_spec_scan_kernel<<<(n + 255) / 256, 256, 0, s>>>(A, e->d_sp_state.p, e->d_sp_app.p, e->d_sp_create.p, e->d_sp_prio.p,
        e->d_sp_gang.p, e->d_sp_cause.p, e->d_atol.p, e->d_aneed.p, e->d_adeny.p, e->d_anode.p, e->d_sp_present.p, P,
        e->d_sp_submit.p, e->nlive, e->d_by_rank.p, e->d_taint.p, e->d_sp_ckey[0].p, e->d_sp_cval[0].p, e->d_sp_pkey[0].p,
        e->d_sp_pval[0].p, e->d_sp_w.p);
    CK(cudaGetLastError());
    size_t tb = e->sp_cub_bytes;
    CK(cub::DeviceRadixSort::SortPairs(e->d_sp_cub.p, tb, e->d_sp_pkey[0].p, e->d_sp_pkey[1].p, e->d_sp_pval[0].p, e->d_sp_pval[1].p, (int)P, 0, 64, s));
    yk_spec_pos_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, e->d_sp_pval[1].p, e->d_sp_pos.p);
    tb = e->sp_cub_bytes;
    CK(cub::DeviceRadixSort::SortPairs(e->d_sp_cub.p, tb, e->d_sp_ckey[0].p, e->d_sp_ckey[1].p, e->d_sp_cval[0].p, e->d_sp_cval[1].p, (int)A, 0, 64, s));
    yk_spec_appkey_kernel<<<(A + 255) / 256, 256, 0, s>>>(A, e->d_sp_cval[1].p, e->d_sp_state.p, e->d_sp_app.p, e->d_sp_cause.p,
                                                         e->d_sp_present.p, e->d_sp_pos.p, P, e->d_sp_ukey[0].p);
    int bits = 1;
    while (bits < 32 && (1ull << bits) <= P) ++bits;
    tb = e->sp_cub_bytes;
    CK(cub::DeviceRadixSort::SortPairs(e->d_sp_cub.p, tb, e->d_sp_ukey[0].p, e->d_sp_ukey[1].p, e->d_sp_cval[1].p, e->d_lt_asks.p, (int)A, 0, bits, s));
    yk_spec_break_kernel<<<(A + 255) / 256, 256, 0, s>>>(A, e->d_lt_asks.p, e->d_sp_sig.p, e->d_sp_w.p, max_bindings, e->d_sp_brk[0].p, e->h_sp_order.d);
    tb = e->sp_cub_bytes;
    CK(cub::DeviceScan::InclusiveSum(e->d_sp_cub.p, tb, e->d_sp_brk[0].p, e->d_sp_brk[1].p, (int)A, s));
    yk_spec_run_kernel<<<(A + 255) / 256, 256, 0, s>>>(A, e->d_sp_brk[1].p, e->un_min, max_bindings, e->d_sp_w.p);
    yk_spec_decide_kernel<<<1, 1, 0, s>>>(e->d_sp_w.p, (uint32_t)e->rd_min, max_bindings, e->h_sp_w.d);
    CK(cudaGetLastError());
    CK(cudaEventRecord(e->ev_sp, s));
    e->st.other_launches += 6 + 3 * 10 + 3;   // six kernels, three cub sorts, one cub scan
    int rc = lt_prepare(e);
    if (rc) return rc;
    ykrd::Args sp{};
    sp.go = e->d_sp_w.p; sp.nan = e->d_flag.p; sp.abort = e->h_sp_abort.d;
    rc = launch_stretch(e, 0, 0, &sp);
    if (rc) return rc;
    e->sp_live = true;
    return YK_OK;
}

// A speculative launch that will not be used: the kernel stops at its next publication, and nothing it wrote is read (the
// next launch or lt_prepare rebuilds records, order and results; its time and passes are never counted).
int spec_discard(yk_engine* e) {
    if (!e->sp_live) return YK_OK;
    e->sp_live = false;
    __atomic_store_n(e->h_sp_abort.p, 1, __ATOMIC_RELEASE);
    const cudaError_t r = cudaStreamSynchronize(e->stream);
    __atomic_store_n(e->h_sp_abort.p, 0, __ATOMIC_RELEASE);
    e->st.spec_discarded++;
    return r == cudaSuccess ? YK_OK : e->cuda_fail(r, "cudaStreamSynchronize (speculative launch)");
}

// After the commit choice: the speculative launch is adopted only when the host's own choice is exactly what it runs -- the
// device commit, planned as one round-eligible stretch over the whole first batch, whose asks equal the device's order
// element for element.  Otherwise it is discarded.
int spec_verify(yk_engine* e, const yklt::Choice& ch) {
    if (!e->sp_live) return YK_OK;
    CK(cudaEventSynchronize(e->ev_sp));
    const uint32_t* w = e->h_sp_w.p;
    const std::vector<uint32_t>& asks = e->slot[0].asks;
    const size_t B = asks.size();
    const std::vector<ykun::Segment>& sg = e->un_segs;
    const bool adopt = ch.device && ch.plan_ready && ch.rounds_only && w[ykspec::W_STATUS] == ykspec::GO && w[ykspec::W_COUNT] == B &&
                       sg.size() == 1 && sg[0].off == 0 && (size_t)sg[0].len == B &&
                       memcmp(asks.data(), e->h_sp_order.p, 4 * B) == 0;
    if (!adopt) return spec_discard(e);
    e->sp_live = false;
    e->sp_adopt = true;
    e->st.spec_adopted++;
    e->st.d2h_bytes += 4 * B;
    return YK_OK;
}

// ---- epochs -------------------------------------------------------------------------------------------
// An epoch is a run of batches swept against ONE sorted view (node order + cap columns as of the epoch start).
// Exactness does not need the view to be fresh: a node not touched since the epoch began has exactly the state
// the view holds, and every touched node is masked out of the bitmaps and handled from the working copy
// (DESIGN.md "ordered commit").  So the order is merged, the availability pushed to the device and the view
// regathered only when the touched set has grown enough to slow the commit down -- and because the sweeps of one
// epoch do not depend on each other's commits, the next batch's sweep and read-back overlap the current commit.
int begin_epoch(yk_engine* e) {
    const int nlive = (int)e->nlive;
    const int Np = (int)round_up((size_t)nlive, NODE_TILE);
    e->epochW = nlive ? Np / 32 : 0;
    e->cm.begin_epoch(e->epochW);
    if (nlive == 0) return YK_OK;
    cudaStream_t s = e->stream;
    CK(cudaMemcpyAsync(e->d_order.p, e->h_order[e->cur].p, sizeof(uint32_t) * (size_t)nlive, cudaMemcpyHostToDevice, s));
    e->st.h2d_bytes += sizeof(uint32_t) * (size_t)nlive;
    yk_gather_kernel<<<(Np + 255) / 256, 256, 0, s>>>(e->D, e->d_total.p, e->d_avail.p, e->maxN, e->d_taint.p, e->d_label.p,
                                                     e->d_flags.p, e->d_order.p, nlive, Np, e->d_scap.p, e->d_staint.p,
                                                     e->d_slabel.p, e->d_snode.p);
    CK(cudaGetLastError());
    e->st.other_launches += 1;
    if (e->ep_rows) {   // every distinct signature of the cycle against the fresh view: one launch, one read-back per epoch
        const int W = e->epochW, WS = W + 1, R = (int)e->ep_n;
        if (!e->ep_uploaded) {
            memcpy(e->ep_h_batch.p, e->ep_reps.data(), sizeof(uint32_t) * (size_t)R);
            CK(cudaMemcpyAsync(e->ep_d_batch.p, e->ep_h_batch.p, sizeof(uint32_t) * (size_t)R, cudaMemcpyHostToDevice, s));
            e->st.h2d_bytes += sizeof(uint32_t) * (size_t)R;
            e->ep_uploaded = true;
        }
        CK(cudaMemset2DAsync(e->ep_d_fit.p + W, sizeof(uint32_t) * (size_t)WS, 0xFF, sizeof(uint32_t), (size_t)R, s));
        CK(cudaEventRecord(e->ep_s0, s));
        YkSweepArgs a{};
        a.s_cap = e->d_scap.p; a.s_taint = e->d_staint.p; a.s_label = e->d_slabel.p; a.s_node = e->d_snode.p; a.Np = Np;
        a.a_req = e->d_areq.p; a.a_tol = e->d_atol.p; a.a_need = e->d_aneed.p; a.a_deny = e->d_adeny.p; a.a_node = e->d_anode.p;
        a.lda = e->maxA; a.batch = e->ep_d_batch.p; a.row0 = 0; a.rows = R;
        a.fit = e->ep_d_fit.p; a.W = W; a.WS = WS; a.n_peer = 0;
        launch_sweep(e->D, a, s, e->slots);
        CK(cudaEventRecord(e->ep_s1, s));
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(e->ep_h_fit.p, e->ep_d_fit.p, sizeof(uint32_t) * (size_t)R * WS, cudaMemcpyDeviceToHost, s));
        CK(cudaEventRecord(e->ep_ev, s));
        e->ep_landed = false;
        e->st.sweep_launches += 1;
        e->st.evaluations += (uint64_t)R * (uint64_t)nlive;
        e->st.rows_swept += (uint64_t)R;
        e->st.d2h_bytes += sizeof(uint32_t) * (size_t)R * WS;
    }
    return YK_OK;
}

// new node order = merge(previous order minus the touched nodes, touched nodes by new key); touched availability
// goes back to the column-major host table and to the device table.  `reorder` false = end of cycle (state only).
int end_epoch(yk_engine* e, bool reorder) {
    const int D = e->D, nlive = (int)e->nlive;
    const int nd = (int)e->cm.dirty_list.size();
    if (!nd) return YK_OK;
    const double t0 = now_ms();
    cudaStream_t s = e->stream;
    if (reorder) {
        e->cm.merge_order(e->h_order[e->cur ^ 1].p, nlive);
        e->cur ^= 1;
    }
    // staging is reused: the previous epoch's upload must have been consumed
    CK(cudaStreamSynchronize(s));
    for (int i0 = 0; i0 < nd; i0 += (int)e->h_dirty_nodes.n) {
        const int cnt = std::min<int>(nd - i0, (int)e->h_dirty_nodes.n);
        for (int i = 0; i < cnt; ++i) {
            const uint32_t n = e->cm.dirty_list[(size_t)(i0 + i)];
            e->h_dirty_nodes[(size_t)i] = n;
            for (int k = 0; k < D; ++k) {
                const int64_t v = e->cm.node(n).avail()[k];
                e->h_dirty_vals[(size_t)k * cnt + i] = v;
                e->n_avail[(size_t)k * e->maxN + n] = v;   // column-major host table stays authoritative between cycles
            }
        }
        CK(cudaMemcpyAsync(e->d_dirty_nodes.p, e->h_dirty_nodes.p, 4 * (size_t)cnt, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(e->d_dirty_vals.p, e->h_dirty_vals.p, 8 * (size_t)cnt * D, cudaMemcpyHostToDevice, s));
        yk_apply_avail_kernel<<<(cnt + 255) / 256, 256, 0, s>>>(D, e->d_avail.p, e->maxN, e->d_dirty_nodes.p, e->d_dirty_vals.p, cnt);
        CK(cudaGetLastError());
        e->st.h2d_bytes += (size_t)cnt * (4 + 8 * D);
        e->st.other_launches += 1;
        if (i0 + cnt < nd) CK(cudaStreamSynchronize(s));
    }
    e->st.host_ms[5] += now_ms() - t0;
    return YK_OK;
}

// Launch the device phase of one batch (already filled into sl.asks): sweep of this rank's rows against the epoch
// view, multi-GPU exchange, chunked read-back with one event per chunk.  Returns without waiting.
int produce(yk_engine* e, Slot& sl, yk_stats_t& st) {
    const int D = e->D;
    const int B = (int)sl.asks.size();
    const int nlive = (int)e->nlive;
    sl.B = B; sl.R = 0; sl.W = e->epochW; sl.rows = 0; sl.nchunks = 0;
    if (B == 0 || nlive == 0) return YK_OK;
    const double t0 = now_ms();
    if (e->ep_rows) {   // the rows of every signature were swept when the epoch began: the batch only points at them
        sl.row_of.resize((size_t)B);
        for (int i = 0; i < B; ++i) sl.row_of[(size_t)i] = e->ep_local[e->a_sigid[sl.asks[(size_t)i]]];
        sl.R = (int)e->ep_n;
        st.batches++;
        st.asks_swept += (uint64_t)B;
        st.host_ms[6] += now_ms() - t0;
        return YK_OK;
    }
    const int W = e->epochW, Np = W * 32, WS = W + 1;
    cudaStream_t s = e->stream;
    // one row per distinct predicate signature in the batch (yk_commit.hpp "shared rows")
    e->share.build(e->cm.t, e->a_sig.data(), sl.asks, e->share_rows, sl.reps, sl.row_of);
    const int R = (int)sl.reps.size();
    sl.R = R;
    memcpy(sl.h_batch.p, sl.reps.data(), sizeof(uint32_t) * (size_t)R);
    CK(cudaMemcpyAsync(sl.d_batch.p, sl.h_batch.p, sizeof(uint32_t) * (size_t)R, cudaMemcpyHostToDevice, s));
    st.h2d_bytes += sizeof(uint32_t) * (size_t)R;
    // this rank's shard of the rows (world == 1: all of them).  A sweep too small to pay for the exchange (shared rows:
    // a few dozen rows per batch) is not split at all: every rank sweeps every row locally and nothing is exchanged.
    // All ranks see the same R and nlive, so they take the same branch.
    const int G = std::max<int>(1, (int)e->cfg.world);
    const bool split = G > 1 && (uint64_t)R * (uint64_t)nlive >= e->split_min_pairs;
    const int world = split ? G : 1;
    const int my_rank = split ? (int)e->cfg.rank : 0;
    const int rows_per = (R + world - 1) / world;
    const int row0 = std::min(R, my_rank * rows_per);
    const int rows = std::min(R, row0 + rows_per) - row0;
    const int Bpad = rows_per * world;
    sl.rows = rows;
    // the last word of every row (first-fit position) starts at YK_NONE
    const int slot_id = (int)(&sl - e->slot);
    const bool p2p_on = G > 1 && e->p2p;   // peers can write into this rank's slots
    const bool p2p = split && p2p_on;      // ... and do, for this batch
    uint32_t value = 0;
    const long long spin_limit = 4000000000ll;   // ~2 s of SM clocks: a dead peer becomes YK_ERR_COMM, not a hang
    if (p2p_on) {
        // The slot's previous content must have been consumed by every rank before anybody overwrites it.  Batches that
        // are not split take part in this hand-shake too (not in the "rows ready" one): ranks are not in lock-step, and
        // a rank that is ahead must not publish the rows of a later, split batch into a slot this rank still reads.
        value = ++e->seq;
        yk_p2p_wait_kernel<<<1, 32, 0, s>>>(e->d_sync.p, G, 16 + slot_id * 8, sl.last_value, e->d_flag.p, spin_limit);
        sl.last_value = value;
        st.other_launches += 1;
    } else {
        // the last word of every row (first-fit position) starts at YK_NONE
        CK(cudaMemset2DAsync(sl.d_fit.p + W, sizeof(uint32_t) * (size_t)WS, 0xFF, sizeof(uint32_t), (size_t)Bpad, s));
    }
    CK(cudaEventRecord(sl.ev_s0, s));
    if (rows > 0) {
        YkSweepArgs a{};
        a.s_cap = e->d_scap.p; a.s_taint = e->d_staint.p; a.s_label = e->d_slabel.p; a.s_node = e->d_snode.p; a.Np = Np;
        a.a_req = e->d_areq.p; a.a_tol = e->d_atol.p; a.a_need = e->d_aneed.p; a.a_deny = e->d_adeny.p; a.a_node = e->d_anode.p;
        a.lda = e->maxA; a.batch = sl.d_batch.p; a.row0 = row0; a.rows = rows;
        a.fit = sl.d_fit.p; a.W = W; a.WS = WS;
        a.n_peer = p2p ? world : 0;
        for (int g = 0; g < 8; ++g) a.fit_peer[g] = p2p && g < world ? e->peer_fit[slot_id][g] : nullptr;
        launch_sweep(D, a, s, e->slots);
        st.sweep_launches += 1;
        st.evaluations += (uint64_t)rows * (uint64_t)nlive;
    }
    CK(cudaEventRecord(sl.ev_s1, s));
    CK(cudaGetLastError());
    if (p2p) {
        YkPeerSync ps{};
        YkPeerFit pf{};
        for (int g = 0; g < world; ++g) { ps.sync[g] = e->peer_sync[g]; pf.fit[g] = e->peer_fit[slot_id][g]; }
        if (rows > 0)
            yk_p2p_first_kernel<<<(rows + 255) / 256, 256, 0, s>>>(sl.d_fit.p, pf, world, my_rank, row0, rows, W, WS);
        yk_p2p_signal_kernel<<<1, 32, 0, s>>>(ps, world, slot_id * 8 + my_rank, value);            // my rows are in place
        yk_p2p_wait_kernel<<<1, 32, 0, s>>>(e->d_sync.p, world, slot_id * 8, value, e->d_flag.p, spin_limit);   // everybody's are
        CK(cudaGetLastError());
        st.other_launches += 3;
    } else if (world > 1) {
        if (!e->xfn) return e->fail(YK_ERR_COMM, "world > 1 but neither a peer-to-peer nor a callback exchange is set up");
        if (e->xfn(e->xctx, sl.d_fit.p, (uint64_t)WS * 4, (uint32_t)row0, (uint32_t)rows_per, (uint32_t)Bpad, (void*)s) != 0)
            return e->fail(YK_ERR_COMM, "exchange callback failed");
    }
    if (p2p_on) CK(cudaMemcpyAsync(sl.h_err.p, e->d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));   // flag waits timed out?
    // read-back in row chunks so the ordered commit overlaps the transfer
    sl.chunk = std::max(128, (R + (int)sl.ev.size() - 1) / (int)sl.ev.size());
    sl.nchunks = (R + sl.chunk - 1) / sl.chunk;
    for (int c = 0; c < sl.nchunks; ++c) {
        const size_t r0 = (size_t)c * sl.chunk, r1 = std::min<size_t>((size_t)R, r0 + sl.chunk);
        CK(cudaMemcpyAsync(sl.h_fit.p + r0 * WS, sl.d_fit.p + r0 * WS, sizeof(uint32_t) * (r1 - r0) * WS, cudaMemcpyDeviceToHost, s));
        CK(cudaEventRecord(sl.ev[(size_t)c], s));
    }
    if (p2p_on) {
        // consumed: wipe the slot (every word back to 0xFFFFFFFF, so first-fit words start at YK_NONE whatever the next
        // row layout is) and tell every rank it may publish into it again
        CK(cudaMemsetAsync(sl.d_fit.p, 0xFF, sl.d_fit.n * sizeof(uint32_t), s));
        YkPeerSync ps{};
        for (int g = 0; g < G; ++g) ps.sync[g] = e->peer_sync[g];
        yk_p2p_signal_kernel<<<1, 32, 0, s>>>(ps, G, 16 + slot_id * 8 + (int)e->cfg.rank, value);
        CK(cudaGetLastError());
        st.other_launches += 1;
    }
    st.d2h_bytes += sizeof(uint32_t) * (size_t)R * WS;
    st.batches++;
    st.asks_swept += (uint64_t)B;
    st.rows_swept += (uint64_t)R;
    st.host_ms[6] += now_ms() - t0;
    return YK_OK;
}

// wait until everything issued for the slot has landed (used before its buffers are reused or it is dropped)
int drain(yk_engine* e, Slot& sl) {
    if (sl.B > 0 && sl.nchunks > 0) CK(cudaEventSynchronize(sl.ev[(size_t)sl.nchunks - 1]));
    return YK_OK;
}

// Ordered commit of one batch from its (arriving) bitmaps: the logic is yk::Committer::commit_batch; this wrapper
// supplies the rows as the read-back chunks land and keeps the timing / counters.  Only called while nodes are live.
int commit(yk_engine* e, Slot& sl, bool insensitive, std::vector<uint32_t>& result, size_t& consumed) {
    const std::vector<uint32_t>& batch = sl.asks;
    if (e->ep_rows) {
        double t_wait = 0;
        const double t1 = now_ms();
        if (!e->ep_landed) {
            const cudaError_t ce = cudaEventSynchronize(e->ep_ev);
            if (ce != cudaSuccess) return e->cuda_fail(ce, "cudaEventSynchronize(epoch rows)");
            e->ep_landed = true;
            t_wait = now_ms() - t1;
            float ms_sweep = 0;
            cudaEventElapsedTime(&ms_sweep, e->ep_s0, e->ep_s1);
            e->st.sweep_ms += ms_sweep;
            e->st.last_sweep_ms = ms_sweep;
            e->st.last_sweep_pairs = (uint64_t)e->ep_n * (uint64_t)e->nlive;
        }
        const int R = sl.R;
        const int rc = e->cm.commit_batch(batch, sl.row_of.data(), e->ep_h_fit.p, insensitive, result, consumed, [R](int) { return R; });
        if (rc == -5) return e->fail(YK_ERR_RANGE, "NaN node score after commit");
        if (rc < 0) return e->fail(YK_ERR_CUDA, "commit aborted");
        const double t2 = now_ms();
        e->st.host_ms[3] += t_wait;
        e->st.host_ms[4] += (t2 - t1) - t_wait;
        e->st.commit_ms += (t2 - t1) - t_wait;
        return YK_OK;
    }
    double t_wait = 0;
    const double t1 = now_ms();
    int next_chunk = 0, wait_rc = YK_OK;
    auto wait = [&](int row) -> int {   // block until the chunk holding `row` has landed; -> rows landed so far
        while (row >= next_chunk * sl.chunk) {
            const double tw = now_ms();
            const cudaError_t ce = cudaEventSynchronize(sl.ev[(size_t)next_chunk]);
            t_wait += now_ms() - tw;
            if (ce != cudaSuccess) { wait_rc = e->cuda_fail(ce, "cudaEventSynchronize(read-back chunk)"); return -1; }
            ++next_chunk;
            if (e->p2p && sl.h_err[0]) {
                wait_rc = e->fail(YK_ERR_COMM, "peer-to-peer exchange timed out waiting for another rank");
                return -1;
            }
        }
        return std::min(sl.R, next_chunk * sl.chunk);
    };
    const int rc = e->cm.commit_batch(batch, sl.row_of.data(), sl.h_fit.p, insensitive, result, consumed, wait);
    if (rc == -5) return e->fail(YK_ERR_RANGE, "NaN node score after commit");
    if (rc < 0) return wait_rc ? wait_rc : e->fail(YK_ERR_CUDA, "commit aborted");
    // all read-back must have landed before the slot's buffers are reused
    {
        const double tw = now_ms();
        { int rcd = drain(e, sl); if (rcd) return rcd; }
        t_wait += now_ms() - tw;
    }
    const double t2 = now_ms();
    e->st.host_ms[3] += t_wait;
    e->st.host_ms[4] += (t2 - t1) - t_wait;
    e->st.commit_ms += (t2 - t1) - t_wait;
    float ms_sweep = 0;
    cudaEventElapsedTime(&ms_sweep, sl.ev_s0, sl.ev_s1);
    e->st.sweep_ms += ms_sweep;
    e->st.last_sweep_ms = ms_sweep;
    e->st.last_sweep_pairs = (uint64_t)sl.rows * (uint64_t)e->nlive;
    return YK_OK;
}

}  // namespace

// ======================================= C ABI =======================================
// idx[] = first, first+1, ... : the bulk-load shape; lets the upserts copy whole columns
static bool contiguous_run(const uint32_t* idx, uint32_t n) {
    for (uint32_t i = 1; i < n; ++i) if (idx[i] != idx[0] + i) return false;
    return n > 0;
}
// Every int64 sum that allocated ask a is counted in, as f(k, sum, sign) for dimension k: its bound node's available
// (sign -1; only while the node is present, and only with `node`), then +1 for every queue on its application's chain, the
// application, and the user-limit entries that apply to the application's user.  The one definition of what an allocation
// is accounted in: alloc_move and alloc_move_fits walk it.
template <typename F>
static void alloc_sums(yk_engine* e, uint32_t a, bool node, F&& f) {
    const uint32_t n = e->a_bound[a], p = e->a_app[a];
    for (int k = 0; k < e->D; ++k) {
        if (node && n != YK_NONE && e->n_present[n]) f(k, e->n_avail[(size_t)k * e->maxN + n], -1);
        for (uint32_t q = e->p_queue[p]; q != YK_NONE; q = e->q_parent[q]) f(k, e->q_alloc[(size_t)k * e->nq + q], +1);
        f(k, e->p_alloc[(size_t)k * e->maxP + p], +1);
    }
    if (!e->n_ul || e->p_user[p] == YK_NONE) return;
    for (uint32_t l = 0; l < e->n_ul; ++l) {
        if (e->ul_user[l] != e->p_user[p]) continue;
        for (uint32_t q = e->p_queue[p]; q != YK_NONE; q = e->q_parent[q])
            if (q == e->ul_queue[l]) {
                for (int k = 0; k < e->D; ++k) f(k, e->ul_alloc[(size_t)k * e->n_ul + l], +1);
                break;
            }
    }
}
// allocated ask a's holdings move by d[0, D): the node's available by -d, the queues, application and user entries by +d
static void alloc_move(yk_engine* e, uint32_t a, const int64_t* d, bool node = true) {
    alloc_sums(e, a, node, [d](int k, int64_t& s, int sign) { s += sign * d[k]; });
}
// whether alloc_move(e, a, d) keeps every sum inside int64
static bool alloc_move_fits(yk_engine* e, uint32_t a, const int64_t* d) {
    bool ok = true;
    alloc_sums(e, a, true, [&](int k, int64_t& s, int sign) {
        int64_t r;
        ok = ok && !(sign > 0 ? __builtin_add_overflow(s, d[k], &r) : __builtin_sub_overflow(s, d[k], &r));
    });
    return ok;
}
// ask x's request is what it is, in d[0, D)
static void ask_request(const yk_engine* e, uint32_t x, int64_t* d) {
    for (int k = 0; k < e->D; ++k) d[k] = e->a_req[(size_t)k * e->maxA + x];
}
// ask x's predicate inputs (request, masks, node) and flags were just rewritten: its signature hash, signature number and
// cause follow.  The number x represented is retired, so asks still holding it stay equal among themselves.
static void ask_resign(yk_engine* e, const yk::CommitTables& sv, uint32_t x) {
    e->a_sig[x] = yk::ask_signature(sv, x);
    e->sigs.retire(x);
    if (e->sigs.n > 2 * e->maxA) {   // too many stale numbers: renumber the present asks
        e->sigs.reset(e->maxA);
        for (uint32_t y = 0; y < e->a_hi; ++y) if (y != x && e->a_state[y] != yk::ST_ABSENT) e->a_sigid[y] = e->sigs.get(sv, e->a_sig[y], y);
    }
    e->a_sigid[x] = e->sigs.get(sv, e->a_sig[x], x);
    e->a_cause[x] = yk::ask_cause(e->D, e->a_req.p, e->maxA, e->a_flags.data(), x);
}
// just enough of a view of the ask tables for the signature hash
static yk::CommitTables sig_view(yk_engine* e) {
    yk::CommitTables sv;
    sv.D = e->D; sv.lda = e->maxA; sv.a_req = e->a_req.p; sv.a_tol = e->a_tol.p; sv.a_need = e->a_need.p; sv.a_deny = e->a_deny.p; sv.a_node = e->a_node.p;
    return sv;
}

template <typename T>
static void copy_or_fill(T* dst, const T* src, uint32_t n, T dflt) {
    if (src) memcpy(dst, src, sizeof(T) * (size_t)n);
    else std::fill(dst, dst + n, dflt);
}

extern "C" {

uint32_t yk_abi_version(void) { return YK_ABI_VERSION; }

const char* yk_strerror(int s) {
    switch (s) {
        case YK_OK: return "ok";
        case YK_ERR_ARG: return "invalid argument";
        case YK_ERR_CUDA: return "CUDA error (no device, no sm_90a image, or launch/copy failure)";
        case YK_ERR_NOMEM: return "out of memory";
        case YK_ERR_STATE: return "invalid state";
        case YK_ERR_RANGE: return "value out of range (NaN node score)";
        case YK_ERR_COMM: return "multi-GPU exchange failed";
        default: return "unknown status";
    }
}

const char* yk_last_error(yk_engine* e) { return e ? e->err.c_str() : "null engine"; }

void yk_destroy(yk_engine* e) {
    if (!e) return;
    e->worker.stop();
    if (e->stream) cudaStreamSynchronize(e->stream);
    if (e->hp_on && e->hp_n)
        fprintf(stderr, "[ykgpu] host ms per cycle (%llu cycles): prologue %.3f  upload+device_order+speculative launch and hints %.3f  wait orderer setup %.3f  "
                        "first fill + commit choice %.3f  verify speculative launch %.3f  run %.3f (of which settling behind the round kernel %.3f)  "
                        "epoch end / export + sync %.3f  finish %.3f\n",
                (unsigned long long)e->hp_n, e->hp[0] / e->hp_n, e->hp[1] / e->hp_n, e->hp[2] / e->hp_n, e->hp[3] / e->hp_n, e->hp[8] / e->hp_n,
                e->hp[4] / e->hp_n, e->hp[7] / e->hp_n, e->hp[5] / e->hp_n, e->hp[6] / e->hp_n);
    if (e->lt_prof && e->d_lt_prof.p) {
        long long pf[32] = {0};
        if (cudaMemcpy(pf, e->d_lt_prof.p, sizeof(pf), cudaMemcpyDeviceToHost) == cudaSuccess) {
            static const char* nm[yklt::PF_N] = {"stage", "scan", "window", "bound", "lattice", "sort", "links+rows", "chain", "apply", "patch", "fullscan"};
            fprintf(stderr, "[ykgpu] lattice kernel, SM clocks per phase (%llu sub-runs):", (unsigned long long)e->lt_total_subruns);
            for (int k = 0; k < yklt::PF_N; ++k) fprintf(stderr, " %s=%lld", nm[k], pf[k]);
            fprintf(stderr, "\n");
            static const char* rn[ykrd::RP_N] = {"stretch_edges", "candidates", "prefix_min", "apply", "sort", "merge", "single_steps"};
            fprintf(stderr, "[ykgpu] round kernel, SM clocks per phase (%llu passes):", (unsigned long long)e->st.round_passes);
            for (int k = 0; k < ykrd::RP_N; ++k) fprintf(stderr, " %s=%lld", rn[k], pf[16 + k]);
            fprintf(stderr, "\n");
        }
    }
    for (int g = 0; g < 8; ++g)
        if (e->peer_open[g]) { cudaIpcCloseMemHandle(e->peer_fit[0][g]); cudaIpcCloseMemHandle(e->peer_fit[1][g]); cudaIpcCloseMemHandle(e->peer_sync[g]); }
    if (e->stream) cudaStreamSynchronize(e->stream);
    if (e->ev0) cudaEventDestroy(e->ev0);
    if (e->ev1) cudaEventDestroy(e->ev1);
    if (e->ev2) cudaEventDestroy(e->ev2);
    if (e->ep_ev) cudaEventDestroy(e->ep_ev);
    if (e->ep_s0) cudaEventDestroy(e->ep_s0);
    if (e->ep_s1) cudaEventDestroy(e->ep_s1);
    if (e->ev_l0) cudaEventDestroy(e->ev_l0);
    if (e->ev_l1) cudaEventDestroy(e->ev_l1);
    if (e->ev_sp) cudaEventDestroy(e->ev_sp);
    for (Slot& sl : e->slot) {
        for (auto ev : sl.ev) if (ev) cudaEventDestroy(ev);
        if (sl.ev_s0) cudaEventDestroy(sl.ev_s0);
        if (sl.ev_s1) cudaEventDestroy(sl.ev_s1);
    }
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

int yk_create(const yk_config* cfg, yk_engine** out) {
    if (!cfg || !out) return YK_ERR_ARG;
    *out = nullptr;
    if (cfg->abi_version != YK_ABI_VERSION || cfg->D < 1 || cfg->D > YK_MAX_D || cfg->policy > 1) return YK_ERR_ARG;
    if (!cfg->max_nodes || !cfg->max_asks || !cfg->max_apps || !cfg->max_queues) return YK_ERR_ARG;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return YK_ERR_CUDA;   // fail loudly: no CPU path
    if (cfg->device >= 0) { if (cudaSetDevice(cfg->device) != cudaSuccess) return YK_ERR_CUDA; }
    yk_engine* e = new (std::nothrow) yk_engine();
    if (!e) return YK_ERR_NOMEM;
    e->cfg = *cfg;
    e->share_rows = !(cfg->flags & YK_FLAG_NO_ROW_SHARING) && !getenv("YK_NO_ROW_SHARING");
    if (const char* sp = getenv("YK_SPLIT_MIN_PAIRS")) e->split_min_pairs = strtoull(sp, nullptr, 10);
    e->D = (int)cfg->D;
    e->maxN = cfg->max_nodes; e->maxA = cfg->max_asks; e->maxP = cfg->max_apps; e->maxQ = cfg->max_queues;
    e->batch = cfg->batch ? cfg->batch : 4096;
    for (int k = 0; k < 8; ++k) e->w.w[k] = k < e->D ? cfg->weights[k] : 0.0;
    const int D = e->D;
    const size_t N = e->maxN, A = e->maxA, Bm = e->batch;
    const size_t Npmax = round_up(N, NODE_TILE);
    e->Wmax = Npmax / 32;
    bool ok = true;
    auto T = [&](cudaError_t r) { if (r != cudaSuccess) { ok = false; e->err = cudaGetErrorString(r); } };
    T(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    T(cudaEventCreate(&e->ev0)); T(cudaEventCreate(&e->ev1)); T(cudaEventCreate(&e->ev2));
    T(e->n_total.alloc(N * D)); T(e->n_avail.alloc(N * D)); T(e->n_taint.alloc(N)); T(e->n_label.alloc(N)); T(e->n_flags.alloc(N));
    T(e->by_rank.alloc(N));
    T(e->a_req.alloc(A * D)); T(e->a_tol.alloc(A)); T(e->a_need.alloc(A)); T(e->a_deny.alloc(A)); T(e->a_node.alloc(A));
    T(e->d_total.alloc(N * D)); T(e->d_avail.alloc(N * D)); T(e->d_taint.alloc(N)); T(e->d_label.alloc(N)); T(e->d_flags.alloc(N));
    T(e->d_by_rank.alloc(N));
    T(e->d_areq.alloc(A * D)); T(e->d_atol.alloc(A)); T(e->d_aneed.alloc(A)); T(e->d_adeny.alloc(A)); T(e->d_anode.alloc(A));
    T(e->d_key_in.alloc(N)); T(e->d_key_out.alloc(N)); T(e->d_val_in.alloc(N)); T(e->d_val_out.alloc(N));
    if (ok) {
        size_t tb = 0;
        T(cub::DeviceRadixSort::SortPairs(nullptr, tb, e->d_key_in.p, e->d_key_out.p, e->d_val_in.p, e->d_val_out.p, (int)N, 0, 64, e->stream));
        e->cub_bytes = tb;
        T(e->d_cub.alloc(tb));
    }
    T(e->d_scap.alloc(Npmax * D)); T(e->d_staint.alloc(Npmax)); T(e->d_slabel.alloc(Npmax)); T(e->d_snode.alloc(Npmax));
    const size_t Bpad = Bm + std::max<uint32_t>(cfg->world, 1);   // rows rounded up to a multiple of world
    T(e->d_flag.alloc(1));
    T(e->h_order[0].alloc(N)); T(e->h_order[1].alloc(N)); T(e->d_order.alloc(N));
    for (Slot& sl : e->slot) {
        T(sl.d_batch.alloc(Bm)); T(sl.d_fit.alloc(Bpad * (e->Wmax + 1)));
        T(sl.h_batch.alloc(Bm)); T(sl.h_fit.alloc(Bm * (e->Wmax + 1))); T(sl.h_err.alloc(1));
        sl.ev.assign(16, nullptr);
        for (auto& ev : sl.ev) T(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        T(cudaEventCreate(&sl.ev_s0)); T(cudaEventCreate(&sl.ev_s1));
    }
    T(e->d_sync.alloc(32));
    if (ok) {
        T(cudaMemset(e->d_sync.p, 0, 32 * sizeof(uint32_t)));
        for (Slot& sl : e->slot) T(cudaMemset(sl.d_fit.p, 0xFF, sl.d_fit.n * sizeof(uint32_t)));
    }
    e->epoch_floor = std::max<uint32_t>(2 * e->batch, 4096);
    if (const char* v = getenv("YK_EPOCH_NODES")) e->epoch_env = (uint32_t)std::max(1, atoi(v));   // tuning / debugging knob
    e->no_spec = getenv("YK_NO_SPECULATION") != nullptr;
    e->prof = getenv("YK_PROFILE_COMMIT") != nullptr;
    if (ok) { int dev = 0; cudaGetDevice(&dev); e->worker.start(dev); }
    T(e->d_dirty_nodes.alloc(N)); T(e->d_dirty_vals.alloc(N * D)); T(e->d_scores.alloc(N));
    // device-resident ordered commit
    e->lt_allowed = !(cfg->flags & YK_FLAG_HOST_COMMIT) && cfg->world <= 1;
    e->lt_auto = true;
    if (cfg->flags & YK_FLAG_DEVICE_COMMIT) e->lt_force = 1;
    e->bp_device = (cfg->flags & YK_FLAG_BINPACKING_DEVICE) != 0;
    if (const char* cm = getenv("YK_COMMIT")) {
        if (!strcmp(cm, "host")) e->lt_allowed = false;
        if (!strcmp(cm, "device")) e->lt_force = 1;
        if (!strcmp(cm, "auto")) { e->lt_auto = true; e->lt_force = 0; e->lt_allowed = !(cfg->flags & YK_FLAG_HOST_COMMIT) && cfg->world <= 1; }
    }
    e->lt_RS = yklt::record_words(D);
    T(e->d_rec.alloc(N * (size_t)e->lt_RS)); T(e->d_ord[0].alloc(N)); T(e->d_ord[1].alloc(N)); T(e->d_rank.alloc(N));
    T(e->d_lt_cur.alloc(1)); T(e->d_lt_hdr.alloc(yklt::H_WORDS)); T(e->d_lt_ub.alloc(8));
    T(e->d_lt_asks.alloc(A)); T(e->d_lt_meta.alloc(A)); T(e->d_lt_shp.alloc(A)); T(e->d_lt_sig.alloc(A)); T(e->d_lt_res.alloc(A));
    T(e->h_lt_asks.alloc(A)); T(e->h_lt_meta.alloc(A)); T(e->h_lt_shp.alloc(A)); T(e->h_lt_sig.alloc(A)); T(e->h_lt_res.alloc(A)); T(e->h_lt_hdr.alloc(yklt::H_WORDS)); T(e->h_lt_ub.alloc(8));
    T(cudaEventCreate(&e->ev_l0)); T(cudaEventCreate(&e->ev_l1));
    T(e->ep_d_batch.alloc(yk_engine::EP_MAX)); T(e->ep_h_batch.alloc(yk_engine::EP_MAX));
    T(e->ep_d_fit.alloc((size_t)yk_engine::EP_MAX * (e->Wmax + 1))); T(e->ep_h_fit.alloc((size_t)yk_engine::EP_MAX * (e->Wmax + 1)));
    T(cudaEventCreateWithFlags(&e->ep_ev, cudaEventDisableTiming)); T(cudaEventCreate(&e->ep_s0)); T(cudaEventCreate(&e->ep_s1));
    e->lt_prof = getenv("YK_PROFILE_LATTICE") != nullptr;
    e->hp_on = getenv("YK_PROFILE_HOST") != nullptr;
    if (const char* um = getenv("YK_UNIFORM_MIN")) e->un_min = atoi(um);   // 0: no uniform-run path
    if (const char* ud = getenv("YK_UNIFORM_DEPTH")) e->un_depth = std::max(0, atoi(ud));   // 0 / unset: the engine's own rule
    if (const char* rm = getenv("YK_ROUND_MIN")) e->rd_min = std::max(0, atoi(rm));         // 0: no cycle starts on the round commit
    if (const char* rw = getenv("YK_ROUND_WINDOW")) e->rd_window = std::max(1, std::min(atoi(rw), ykrd::WCAP));
    if (const char* rg = getenv("YK_ROUND_GUARD")) e->rd_guard = std::max(0, atoi(rg));
    T(e->d_rd_spent.alloc(N)); T(e->d_rd_req.alloc(A * (size_t)D)); T(e->d_rd_hdr.alloc(ykrd::R_WORDS)); T(e->h_rd_hdr.alloc(ykrd::R_WORDS));
    T(e->h_rd_res.alloc(A, true)); T(e->h_rd_prog.alloc(1, true));
    T(e->d_sp_app.alloc(A)); T(e->d_sp_gang.alloc(A)); T(e->d_sp_sig.alloc(A)); T(e->d_sp_create.alloc(A)); T(e->d_sp_prio.alloc(A));
    T(e->d_sp_cause.alloc(A)); T(e->d_sp_state.alloc(A)); T(e->d_sp_submit.alloc(e->maxP)); T(e->d_sp_present.alloc(e->maxP));
    for (int b = 0; b < 2; ++b) {
        T(e->d_sp_ckey[b].alloc(A)); T(e->d_sp_cval[b].alloc(A)); T(e->d_sp_ukey[b].alloc(A)); T(e->d_sp_brk[b].alloc(A));
        T(e->d_sp_pkey[b].alloc(e->maxP)); T(e->d_sp_pval[b].alloc(e->maxP));
    }
    T(e->d_sp_pos.alloc(e->maxP)); T(e->d_sp_w.alloc(ykspec::W_N));
    T(e->h_sp_state.alloc(A)); T(e->h_sp_order.alloc(A, true)); T(e->h_sp_w.alloc(ykspec::W_N, true)); T(e->h_sp_init.alloc(ykspec::W_N));
    T(e->h_sp_abort.alloc(1, true));
    T(cudaEventCreateWithFlags(&e->ev_sp, cudaEventDisableTiming));
    if (ok) {
        size_t b1 = 0, b2 = 0, b3 = 0, b4 = 0;
        T(cub::DeviceRadixSort::SortPairs(nullptr, b1, e->d_sp_ckey[0].p, e->d_sp_ckey[1].p, e->d_sp_cval[0].p, e->d_sp_cval[1].p, (int)A, 0, 64, e->stream));
        T(cub::DeviceRadixSort::SortPairs(nullptr, b2, e->d_sp_pkey[0].p, e->d_sp_pkey[1].p, e->d_sp_pval[0].p, e->d_sp_pval[1].p, (int)e->maxP, 0, 64, e->stream));
        T(cub::DeviceRadixSort::SortPairs(nullptr, b3, e->d_sp_ukey[0].p, e->d_sp_ukey[1].p, e->d_sp_cval[1].p, e->d_lt_asks.p, (int)A, 0, 32, e->stream));
        T(cub::DeviceScan::InclusiveSum(nullptr, b4, e->d_sp_brk[0].p, e->d_sp_brk[1].p, (int)A, e->stream));
        e->sp_cub_bytes = std::max(std::max(b1, b2), std::max(b3, b4));
        T(e->d_sp_cub.alloc(e->sp_cub_bytes));
        e->h_sp_init[ykspec::W_PRIO_MIN] = 0xFFFFFFFFu;   // every other word starts at 0
    }
    T(e->d_lt_prof.alloc(32));   // [0, 16) the lattice kernel's phases, [16, 32) the round kernel's
    if (ok) T(cudaMemset(e->d_lt_prof.p, 0, 32 * sizeof(long long)));
    if (ok) T(lattice_setup(D, &e->lt_smem));
    if (ok) T(rounds_setup(D, &e->rd_smem));
    T(e->h_snode.alloc(N)); T(e->h_skey.alloc(N));
    T(e->h_dirty_nodes.alloc(N)); T(e->h_dirty_vals.alloc(N * D)); T(e->h_flag.alloc(1)); T(e->h_scores.alloc(N));
    if (ok) {   // does this binary carry an image the device can run?
        cudaFuncAttributes fa;
        T(cudaFuncGetAttributes(&fa, yk_key_kernel));
        int dev = 0, sms = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        e->slots = sweep_slots(D, sms);
    }
    if (!ok) { yk_destroy(e); return YK_ERR_CUDA; }
    e->n_rank.assign(N, 0); e->n_present.assign(N, 0);
    e->a_shape.assign(A, 0); e->a_sigid.assign(A, 0); e->a_cause.assign(A, 0);
    e->sigs.reset(A);
    e->a_sig.assign(A, 0); e->a_prio.assign(A, 0); e->a_create.assign(A, 0); e->a_app.assign(A, 0); e->a_flags.assign(A, 0);
    e->a_gang.assign(A, YK_NONE); e->a_bound.assign(A, YK_NONE); e->a_state.assign(A, yk::ST_ABSENT);
    e->pp_mark.assign(A, 0); e->pp_plan.assign(A, YK_NONE);
    e->p_queue.assign(e->maxP, 0); e->p_submit.assign(e->maxP, 0); e->p_present.assign(e->maxP, 0); e->p_user.assign(e->maxP, YK_NONE);
    e->p_alloc.assign((size_t)e->maxP * D, 0);
    // default queue tree: root only would have no leaf for apps; root + one leaf "root.default"
    e->nq = 0;
    
    *out = e;
    return YK_OK;
}

int yk_nodes_upsert(yk_engine* e, uint32_t n, const uint32_t* idx, const int64_t* total, const int64_t* avail,
                    const uint64_t* taint, const uint64_t* label, const uint32_t* name_rank, const uint32_t* flags) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!idx || !total || !avail || !name_rank)) return e->fail(YK_ERR_ARG, "yk_nodes_upsert: null array");
    for (uint32_t i = 0; i < n; ++i) if (idx[i] >= e->maxN) return e->fail(YK_ERR_ARG, "yk_nodes_upsert: index beyond max_nodes");
    if (contiguous_run(idx, n)) {   // whole-column copies
        const uint32_t x0 = idx[0];
        for (int k = 0; k < e->D; ++k) {
            memcpy(&e->n_total[(size_t)k * e->maxN + x0], total + (size_t)k * n, sizeof(int64_t) * (size_t)n);
            memcpy(&e->n_avail[(size_t)k * e->maxN + x0], avail + (size_t)k * n, sizeof(int64_t) * (size_t)n);
        }
        copy_or_fill<uint64_t>(&e->n_taint[x0], taint, n, 0);
        copy_or_fill<uint64_t>(&e->n_label[x0], label, n, 0);
        copy_or_fill<uint32_t>(&e->n_flags[x0], flags, n, YK_NODE_SCHEDULABLE);
        for (uint32_t i = 0; i < n && !e->rank_stale; ++i)
            if (!e->n_present[x0 + i] || e->n_rank[x0 + i] != name_rank[i]) e->rank_stale = true;
        memcpy(&e->n_rank[x0], name_rank, sizeof(uint32_t) * (size_t)n);
        std::fill(e->n_present.begin() + x0, e->n_present.begin() + x0 + n, 1);
        e->n_hi = std::max(e->n_hi, x0 + n);
        e->nodes_stale = true;
        return YK_OK;
    }
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t x = idx[i];
        for (int k = 0; k < e->D; ++k) {
            e->n_total[(size_t)k * e->maxN + x] = total[(size_t)k * n + i];
            e->n_avail[(size_t)k * e->maxN + x] = avail[(size_t)k * n + i];
        }
        e->n_taint[x] = taint ? taint[i] : 0;
        e->n_label[x] = label ? label[i] : 0;
        e->n_flags[x] = flags ? flags[i] : YK_NODE_SCHEDULABLE;
        if (!e->n_present[x] || e->n_rank[x] != name_rank[i]) e->rank_stale = true;
        e->n_rank[x] = name_rank[i];
        e->n_present[x] = 1;
        e->n_hi = std::max(e->n_hi, x + 1);
    }
    e->nodes_stale = true;
    return YK_OK;
}

int yk_nodes_remove(yk_engine* e, uint32_t n, const uint32_t* idx) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && !idx) return e->fail(YK_ERR_ARG, "yk_nodes_remove: null array");
    for (uint32_t i = 0; i < n; ++i) {
        if (idx[i] >= e->maxN) return e->fail(YK_ERR_ARG, "yk_nodes_remove: index beyond max_nodes");
        if (e->n_present[idx[i]]) { e->n_present[idx[i]] = 0; e->n_flags[idx[i]] = 0; e->rank_stale = true; e->nodes_stale = true; }
    }
    return YK_OK;
}

int yk_queues_set(yk_engine* e, uint32_t q, const uint32_t* parent, const int64_t* guaranteed, const int64_t* max,
                  const int64_t* allocated, const uint8_t* sort) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (!q || q > e->maxQ || !parent) return e->fail(YK_ERR_ARG, "yk_queues_set: bad queue count");
    if (parent[0] != YK_NONE) return e->fail(YK_ERR_ARG, "yk_queues_set: queue 0 must be the root");
    for (uint32_t i = 1; i < q; ++i) if (parent[i] >= i) return e->fail(YK_ERR_ARG, "yk_queues_set: parent[i] must be < i");
    const int D = e->D;
    // applications keep pointing at queue indices: a tree that no longer has them (or turned their leaf into a parent) is
    // refused rather than silently re-homing them
    for (uint32_t p = 0; p < e->maxP; ++p) {
        if (!e->p_present[p]) continue;
        if (e->p_queue[p] >= q) return e->fail(YK_ERR_STATE, "yk_queues_set: an application sits in a queue the new tree does not have (remove or move it first)");
        for (uint32_t i = 1; i < q; ++i)
            if (parent[i] == e->p_queue[p]) return e->fail(YK_ERR_STATE, "yk_queues_set: an application sits in a queue the new tree makes a parent");
    }
    e->nq = q;
    e->q_parent.assign(parent, parent + q);
    e->q_guar.assign((size_t)q * D, -1); e->q_max.assign((size_t)q * D, -1); e->q_alloc.assign((size_t)q * D, 0);
    if (guaranteed) e->q_guar.assign(guaranteed, guaranteed + (size_t)q * D);
    if (max) e->q_max.assign(max, max + (size_t)q * D);
    if (allocated) e->q_alloc.assign(allocated, allocated + (size_t)q * D);
    else   // what the present applications hold stays accounted: their allocations are summed up the new tree
        for (uint32_t p = 0; p < e->maxP; ++p) {
            if (!e->p_present[p]) continue;
            for (uint32_t qq = e->p_queue[p]; qq != YK_NONE; qq = e->q_parent[qq])
                for (int k = 0; k < D; ++k) e->q_alloc[(size_t)k * q + qq] += e->p_alloc[(size_t)k * e->maxP + p];
        }
    e->q_sort.assign(q, 0);
    if (sort) e->q_sort.assign(sort, sort + q);
    e->q_prio_offset.assign(q, 0); e->q_prio_fence.assign(q, 0);   // defaults; yk_queues_priority sets them
    e->q_pp_fence.assign(q, 0);                                      // yk_queues_preemption sets it
    for (uint32_t i = 0; i < q; ++i)
        if (e->q_sort[i] > 1) return e->fail(YK_ERR_ARG, "yk_queues_set: unknown application sort policy");
    return YK_OK;
}

int yk_queues_priority(yk_engine* e, uint32_t q, const int32_t* offset, const uint8_t* fence) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (q != e->nq) return e->fail(YK_ERR_ARG, "yk_queues_priority: queue count differs from yk_queues_set");
    e->q_prio_offset.assign(q, 0); e->q_prio_fence.assign(q, 0);
    if (offset) e->q_prio_offset.assign(offset, offset + q);
    if (fence) for (uint32_t i = 0; i < q; ++i) e->q_prio_fence[i] = fence[i] ? 1 : 0;
    return YK_OK;
}

int yk_queues_preemption(yk_engine* e, uint32_t q, const uint8_t* fence) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (q != e->nq) return e->fail(YK_ERR_ARG, "yk_queues_preemption: queue count differs from yk_queues_set");
    e->q_pp_fence.assign(q, 0);
    if (fence) for (uint32_t i = 0; i < q; ++i) e->q_pp_fence[i] = fence[i] ? 1 : 0;
    return YK_OK;
}

int yk_apps_upsert(yk_engine* e, uint32_t n, const uint32_t* idx, const uint32_t* queue, const int64_t* submit) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!idx || !queue || !submit)) return e->fail(YK_ERR_ARG, "yk_apps_upsert: null array");
    for (uint32_t i = 0; i < n; ++i) {
        if (idx[i] >= e->maxP) return e->fail(YK_ERR_ARG, "yk_apps_upsert: index beyond max_apps");
        if (queue[i] >= e->nq) return e->fail(YK_ERR_ARG, "yk_apps_upsert: unknown queue (call yk_queues_set first)");
    }
    // an allocation stays accounted to its application's index and queue chain until it is released: an entry that would
    // zero an index's holdings (it comes back) or move them to another chain is refused while an allocated ask belongs to it
    bool moves = false;
    for (uint32_t i = 0; i < n && !moves; ++i) moves = !e->p_present[idx[i]] || e->p_queue[idx[i]] != queue[i];
    if (moves) {
        std::vector<uint8_t> holds(e->maxP, 0);
        for (uint32_t a = 0; a < e->a_hi; ++a) if (e->a_state[a] == yk::ST_ALLOCATED) holds[e->a_app[a]] = 1;
        for (uint32_t i = 0; i < n; ++i) {
            if (!holds[idx[i]]) continue;
            if (!e->p_present[idx[i]]) return e->fail(YK_ERR_STATE, "yk_apps_upsert: a removed application's index still holds allocations (release them first)");
            if (e->p_queue[idx[i]] != queue[i]) return e->fail(YK_ERR_STATE, "yk_apps_upsert: an application that holds allocations cannot move to another queue");
        }
    }
    for (uint32_t i = 0; i < n; ++i) {
        if (!e->p_present[idx[i]]) for (int k = 0; k < e->D; ++k) e->p_alloc[(size_t)k * e->maxP + idx[i]] = 0;
        e->p_queue[idx[i]] = queue[i]; e->p_submit[idx[i]] = submit[i]; e->p_present[idx[i]] = 1;
    }
    if (n) e->sp_apps_stale = true;
    return YK_OK;
}

int yk_apps_user(yk_engine* e, uint32_t n, const uint32_t* idx, const uint32_t* user) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!idx || !user)) return e->fail(YK_ERR_ARG, "yk_apps_user: null array");
    for (uint32_t i = 0; i < n; ++i) if (idx[i] >= e->maxP) return e->fail(YK_ERR_ARG, "yk_apps_user: index beyond max_apps");
    for (uint32_t i = 0; i < n; ++i) e->p_user[idx[i]] = user[i];
    return YK_OK;
}

int yk_user_limits_set(yk_engine* e, uint32_t n, const uint32_t* queue, const uint32_t* user, const int64_t* max, const int64_t* held) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!queue || !user || !max)) return e->fail(YK_ERR_ARG, "yk_user_limits_set: null array");
    for (uint32_t i = 0; i < n; ++i) if (queue[i] >= e->nq) return e->fail(YK_ERR_ARG, "yk_user_limits_set: unknown queue (call yk_queues_set first)");
    const int D = e->D;
    e->n_ul = n;
    e->ul_queue.assign(queue, queue + n); e->ul_user.assign(user, user + n);
    e->ul_max.assign(max, max + (size_t)n * D);
    if (held) e->ul_alloc.assign(held, held + (size_t)n * D); else e->ul_alloc.assign((size_t)n * D, 0);
    return YK_OK;
}

int yk_apps_remove(yk_engine* e, uint32_t n, const uint32_t* idx) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && !idx) return e->fail(YK_ERR_ARG, "yk_apps_remove: null array");
    for (uint32_t i = 0; i < n; ++i) {
        if (idx[i] >= e->maxP) return e->fail(YK_ERR_ARG, "yk_apps_remove: index beyond max_apps");
        e->p_present[idx[i]] = 0;
    }
    if (n) e->sp_apps_stale = true;
    return YK_OK;
}

int yk_asks_upsert(yk_engine* e, uint32_t a, const uint32_t* idx, const int64_t* req, const uint64_t* tol,
                   const uint64_t* need, const uint64_t* deny, const int32_t* prio, const int64_t* create_seq,
                   const uint32_t* app, const uint32_t* required_node, const uint32_t* flags, const uint32_t* gang) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (a && (!idx || !req || !create_seq || !app)) return e->fail(YK_ERR_ARG, "yk_asks_upsert: null array");
    for (uint32_t i = 0; i < a; ++i) {
        if (idx[i] >= e->maxA) return e->fail(YK_ERR_ARG, "yk_asks_upsert: index beyond max_asks");
        if (app[i] >= e->maxP || !e->p_present[app[i]]) return e->fail(YK_ERR_ARG, "yk_asks_upsert: unknown application");
        if (required_node && required_node[i] != YK_NONE && required_node[i] >= e->maxN)
            return e->fail(YK_ERR_ARG, "yk_asks_upsert: required_node beyond max_nodes");
        if (e->a_state[idx[i]] == yk::ST_ALLOCATED) return e->fail(YK_ERR_STATE, "yk_asks_upsert: ask holds an allocation (release it first)");
    }
    for (uint32_t i = 0; i < a; ++i) e->pp_plan[idx[i]] = YK_NONE;   // a new ask: an earlier plan for the index is gone
    const yk::CommitTables sv = sig_view(e);
    if (contiguous_run(idx, a)) {   // whole-column copies, then the signature hashes in one sequential pass
        const uint32_t x0 = idx[0];
        for (int k = 0; k < e->D; ++k) memcpy(&e->a_req[(size_t)k * e->maxA + x0], req + (size_t)k * a, sizeof(int64_t) * (size_t)a);
        copy_or_fill<uint64_t>(&e->a_tol[x0], tol, a, 0);
        copy_or_fill<uint64_t>(&e->a_need[x0], need, a, 0);
        copy_or_fill<uint64_t>(&e->a_deny[x0], deny, a, 0);
        copy_or_fill<uint32_t>(&e->a_node[x0], required_node, a, YK_NONE);
        copy_or_fill<int32_t>(&e->a_prio[x0], prio, a, 0);
        memcpy(&e->a_create[x0], create_seq, sizeof(int64_t) * (size_t)a);
        memcpy(&e->a_app[x0], app, sizeof(uint32_t) * (size_t)a);
        copy_or_fill<uint32_t>(&e->a_flags[x0], flags, a, 0);
        copy_or_fill<uint32_t>(&e->a_gang[x0], gang, a, YK_NONE);
        std::fill(e->a_state.begin() + x0, e->a_state.begin() + x0 + a, (uint8_t)yk::ST_PENDING);
        std::fill(e->a_bound.begin() + x0, e->a_bound.begin() + x0 + a, YK_NONE);
        // (the rows [x0, x0+a) were overwritten above: numbers they represented are retired first)
        const bool full = x0 == 0 && a >= e->a_hi;
        if (full) e->sigs.reset(e->maxA);
        else for (uint32_t i = 0; i < a; ++i) e->sigs.retire(x0 + i);
        for (uint32_t i = 0; i < a; ++i) e->a_sig[x0 + i] = yk::ask_signature(sv, x0 + i);
        for (uint32_t i = 0; i < a; ++i) e->a_cause[x0 + i] = yk::ask_cause(e->D, e->a_req.p, e->maxA, e->a_flags.data(), x0 + i);
        e->a_hi = std::max(e->a_hi, x0 + a);
        if (!full && e->sigs.n > 2 * e->maxA) {   // too many stale numbers: renumber every present ask
            e->sigs.reset(e->maxA);
            for (uint32_t y = 0; y < e->a_hi; ++y) if (e->a_state[y] != yk::ST_ABSENT) e->a_sigid[y] = e->sigs.get(sv, e->a_sig[y], y);
        } else {
            for (uint32_t i = 0; i < a; ++i) e->a_sigid[x0 + i] = e->sigs.get(sv, e->a_sig[x0 + i], x0 + i);
        }
        e->asks_stale = true;
        return YK_OK;
    }
    for (uint32_t i = 0; i < a; ++i) {
        const uint32_t x = idx[i];
        for (int k = 0; k < e->D; ++k) e->a_req[(size_t)k * e->maxA + x] = req[(size_t)k * a + i];
        e->a_tol[x] = tol ? tol[i] : 0;
        e->a_need[x] = need ? need[i] : 0;
        e->a_deny[x] = deny ? deny[i] : 0;
        e->a_node[x] = required_node ? required_node[i] : YK_NONE;
        e->a_prio[x] = prio ? prio[i] : 0;
        e->a_create[x] = create_seq[i];
        e->a_app[x] = app[i];
        e->a_flags[x] = flags ? flags[i] : 0;
        e->a_gang[x] = gang ? gang[i] : YK_NONE;
        e->a_state[x] = yk::ST_PENDING;
        e->a_bound[x] = YK_NONE;
        e->a_hi = std::max(e->a_hi, x + 1);
        ask_resign(e, sv, x);
    }
    e->asks_stale = true;
    return YK_OK;
}

int yk_asks_remove(yk_engine* e, uint32_t a, const uint32_t* idx) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (a && !idx) return e->fail(YK_ERR_ARG, "yk_asks_remove: null array");
    for (uint32_t i = 0; i < a; ++i) {
        if (idx[i] >= e->maxA) return e->fail(YK_ERR_ARG, "yk_asks_remove: index beyond max_asks");
        if (e->a_state[idx[i]] == yk::ST_ALLOCATED) return e->fail(YK_ERR_STATE, "yk_asks_remove: ask holds an allocation (use yk_release)");
    }
    for (uint32_t i = 0; i < a; ++i) { e->a_state[idx[i]] = yk::ST_ABSENT; e->pp_plan[idx[i]] = YK_NONE; }
    return YK_OK;
}

int yk_release(yk_engine* e, uint32_t n, const uint32_t* idx) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && !idx) return e->fail(YK_ERR_ARG, "yk_release: null array");
    for (uint32_t i = 0; i < n; ++i)
        if (idx[i] >= e->maxA || e->a_state[idx[i]] != yk::ST_ALLOCATED) return e->fail(YK_ERR_STATE, "yk_release: ask holds no allocation");
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t a = idx[i];
        int64_t d[8];
        ask_request(e, a, d);
        for (int k = 0; k < e->D; ++k) d[k] = -d[k];
        alloc_move(e, a, d);
        e->a_state[a] = yk::ST_ABSENT;
        e->a_bound[a] = YK_NONE;
        e->pp_mark[a] = 0;
    }
    e->nodes_stale = true;
    return YK_OK;
}

int yk_asks_resize(yk_engine* e, uint32_t n, const uint32_t* idx, const int64_t* req) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!idx || !req)) return e->fail(YK_ERR_ARG, "yk_asks_resize: null array");
    const int D = e->D;
    std::vector<uint32_t> sorted(idx, idx + n);
    std::sort(sorted.begin(), sorted.end());
    for (uint32_t i = 0; i < n; ++i) {
        if (sorted[i] >= e->maxA) return e->fail(YK_ERR_ARG, "yk_asks_resize: index beyond max_asks");
        if (i && sorted[i] == sorted[i - 1]) return e->fail(YK_ERR_ARG, "yk_asks_resize: the same ask twice");
    }
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t x = idx[i];
        if (e->a_state[x] == yk::ST_ABSENT) return e->fail(YK_ERR_STATE, "yk_asks_resize: ask not present");
        if (e->a_state[x] == yk::ST_ALLOCATED)
            for (int k = 0; k < D; ++k)
                if (req[(size_t)k * n + i] < 0) return e->fail(YK_ERR_ARG, "yk_asks_resize: negative request for an allocated ask");
    }
    // allocations first: each moves by new - old, checked against overflow before it is applied; on an overflow the ones
    // already moved are moved back (exact: they return to the values they had), so nothing has changed
    std::vector<int64_t> delta((size_t)n * D);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t x = idx[i];
        if (e->a_state[x] != yk::ST_ALLOCATED) continue;
        int64_t* d = &delta[(size_t)i * D];
        for (int k = 0; k < D; ++k) d[k] = req[(size_t)k * n + i] - e->a_req[(size_t)k * e->maxA + x];   // both >= 0
        if (alloc_move_fits(e, x, d)) { alloc_move(e, x, d); continue; }
        for (uint32_t j = i; j-- > 0;) {
            if (e->a_state[idx[j]] != yk::ST_ALLOCATED) continue;
            int64_t back[8];
            for (int k = 0; k < D; ++k) back[k] = -delta[(size_t)j * D + k];
            alloc_move(e, idx[j], back);
        }
        return e->fail(YK_ERR_RANGE, "yk_asks_resize: a node's available or a queue's, application's or user's allocation would overflow int64");
    }
    // then the requests; an ask whose vector changed is signed again and gets its cause from the new request
    const yk::CommitTables sv = sig_view(e);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t x = idx[i];
        bool same = true;
        for (int k = 0; k < D; ++k) {
            int64_t& r = e->a_req[(size_t)k * e->maxA + x];
            same = same && r == req[(size_t)k * n + i];
            r = req[(size_t)k * n + i];
        }
        if (!same) ask_resign(e, sv, x);
        e->pp_plan[x] = YK_NONE;
    }
    if (n) e->nodes_stale = e->asks_stale = true;
    return YK_OK;
}

}  // extern "C" (reopened after yk_cycle)

// ---- one cycle ---------------------------------------------------------------------------------------------------
namespace {

// How many distinct signatures do the cycle's pending asks (in index order) have?  Few: every one is swept once per epoch
// (ep_local = its row), no per-batch device work at all
void epoch_rows(yk_engine* e, const std::vector<uint32_t>& pend) {
    e->ep_rows = false;
    if (!e->share_rows || e->cfg.world > 1 || getenv("YK_NO_EPOCH_ROWS")) return;
    if (e->ep_seen.size() < e->sigs.n) { e->ep_seen.assign(e->sigs.n + 1024, 0); e->ep_local.assign(e->sigs.n + 1024, 0); e->ep_stamp = 0; }
    if (++e->ep_stamp == 0) { std::fill(e->ep_seen.begin(), e->ep_seen.end(), 0); e->ep_stamp = 1; }
    e->ep_reps.clear();
    uint32_t ns = 0;
    for (uint32_t a : pend) {
        const uint32_t id = e->a_sigid[a];
        if (e->ep_seen[id] != e->ep_stamp) {
            e->ep_seen[id] = e->ep_stamp;
            if (ns < yk_engine::EP_MAX) { e->ep_local[id] = ns; e->ep_reps.push_back(a); }
            if (++ns > yk_engine::EP_MAX) break;
        }
    }
    e->ep_rows = ns > 0 && ns <= yk_engine::EP_MAX && (uint64_t)ns * 8 <= pend.size();
    e->ep_n = ns;
}

struct Cycle {
    uint32_t max_bindings = 0;
    yk_binding* out = nullptr;
    uint32_t n = 0;                 // bindings so far
    std::vector<uint32_t> result;
};

// one binding: out to the caller, and remembered for yk_release
void bind_one(yk_engine* e, Cycle& c, uint32_t a, uint32_t node) {
    e->a_bound[a] = node;
    c.out[c.n].ask = a; c.out[c.n].node = node;
    ++c.n;
}

// The cycle on the device commit.  slot[0] already holds the first batch (yklt::choose_commit).  Returns with handoff =
// true when the rest of the cycle belongs to the host commit.
int run_lattice(yk_engine* e, Cycle& c, yklt::Choice& ch, bool& handoff) {
    handoff = false;
    int rc = e->sp_adopt ? YK_OK : lt_prepare(e);   // an adopted speculative launch runs on what spec_launch prepared
    if (rc) return rc;
    Slot& A = e->slot[0];
    yklt::Loop lp{e->ord, e->cm.t, ch.shape_ids, e->a_sigid.data(), A.asks, A.snap, c.result,
                  e->h_lt_meta.p, e->h_lt_shp.p, e->h_lt_sig.p, e->un_segs, ch.plan_ready,
                  yklt::min_run(e->cfg.policy == YK_POLICY_BINPACKING, e->un_min), e->nlive == 0,
                  e->ord.insensitive ? (size_t)e->maxA : (size_t)e->batch, c.max_bindings, c.n, e->st};
    if (e->nlive && !A.asks.empty()) {   // the initial order's NaN flag (device_order) is checked before the first batch
                                          // commits anything: a failed cycle must leave the node tables as they were
        // (an adopted launch is still running: the flag landed before the screen's event, and the kernel did nothing on NaN)
        if (e->sp_adopt) CK(cudaEventSynchronize(e->ev_sp));
        else CK(cudaStreamSynchronize(e->stream));
        if (e->h_flag[0]) return e->fail(YK_ERR_RANGE, "NaN node score (zero total on a weighted resource)");
    }
    auto bind = [&](uint32_t a, uint32_t node) { bind_one(e, c, a, node); };
    auto ahead = [&](const uint32_t* res, size_t off, size_t to) { yklt::settle_ahead(lp, res, off, to, bind); };
    auto batch = [&](size_t B, int* status, size_t* consumed) {
        const int rcb = lt_batch(e, B, status, consumed, c.result, ahead);
        if (rcb || *status == yklt::ST_NAN) yklt::settle_back(lp, [&](uint32_t a) { e->a_bound[a] = YK_NONE; --c.n; });
        return rcb;
    };
    return yklt::device_commit(lp, batch, bind, [&](int code, const char* m) { return e->fail(code, m); }, handoff);
}

// The cycle on the sweep + host commit path.  slot[0] holds the first batch (filled, not yet launched); the host commit's
// working copy and the epoch view are set up here.
int run_host(yk_engine* e, Cycle& c) {
    int rc = initial_order(e);
    if (rc) return rc;
    e->cm.set_pending(e->pending);   // smallest pending request per dimension: nodes below it are retired from the walk
    // epoch length: long enough that order merges / view refreshes (and the pipeline bubble they cost) stay rare on big
    // clusters, short enough that the touched set does not slow the walk: 5/8 of the nodes, at least two batches
    e->epoch_limit = e->epoch_env ? e->epoch_env : std::max<uint32_t>(e->epoch_floor, (uint32_t)((uint64_t)e->nlive * 5 / 8));
    // Few-signature cycles (epoch rows) under the fair sort, no gangs: the sweeps cost nothing per batch, so what an epoch end buys
    // (a shorter touched index) is worth less than what it costs (order merge, view refresh, a pipeline bubble): measured on
    // config 2, 6.5 -> 5.8 ms with one epoch for the whole cycle; gang cycles (roll-backs walk the touched index) lose.
    if (!e->epoch_env && e->ep_rows && !e->cycle_has_gang && e->cfg.policy == YK_POLICY_FAIR)
        e->epoch_limit = std::max<uint32_t>(e->epoch_limit, 2u * e->nlive);
    rc = begin_epoch(e);
    if (rc) return rc;
    yk::HostLoop lp{e->ord, c.result, e->nlive == 0, (size_t)e->batch, e->epoch_limit, e->cm.dirty_list, !e->no_spec,
                    c.max_bindings, c.n, e->st, e->wst};
    // the speculated fill and launch run on the helper thread into e->wst, merged at the join
    auto join = [&] {
        e->worker.wait();
        yk_stats_t& w = e->wst;
        e->st.h2d_bytes += w.h2d_bytes; e->st.d2h_bytes += w.d2h_bytes; e->st.batches += w.batches;
        e->st.asks_swept += w.asks_swept; e->st.rows_swept += w.rows_swept;
        e->st.sweep_launches += w.sweep_launches; e->st.evaluations += w.evaluations; e->st.other_launches += w.other_launches;
        e->st.host_ms[7] += w.host_ms[2] + w.host_ms[6];   // orderer + launch time hidden behind the commit
        w = yk_stats_t{};
    };
    return yk::host_commit(lp, e->slot,
                           [&](Slot& sl, yk_stats_t& st) { return produce(e, sl, st); },
                           [&](Slot& sl, std::vector<uint32_t>& result, size_t& consumed) { return commit(e, sl, e->ord.insensitive, result, consumed); },
                           [&](auto&& job) { e->worker.submit(job); }, join,
                           [&](Slot& sl) { return drain(e, sl); },
                           [&] { const int rce = end_epoch(e, true); return rce ? rce : begin_epoch(e); },
                           [&](uint32_t a, uint32_t node) { bind_one(e, c, a, node); },
                           [&](int code, const char* m) { return e->fail(code, m); });
}

}  // namespace

extern "C" int yk_cycle(yk_engine* e, uint32_t max_bindings, yk_binding* out, uint32_t* n_out, uint32_t* slow, uint32_t slow_cap,
             uint32_t* n_slow) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (!n_out || (max_bindings && !out)) return e->fail(YK_ERR_ARG, "yk_cycle: null output");
    *n_out = 0;
    if (n_slow) *n_slow = 0;
    if (e->nq == 0) return e->fail(YK_ERR_STATE, "yk_cycle: no queues configured (yk_queues_set)");
    for (uint32_t p = 0; p < e->maxP; ++p)
        if (e->p_present[p] && e->p_queue[p] >= e->nq) return e->fail(YK_ERR_STATE, "yk_cycle: an application sits in a queue that no longer exists");
    const double t_start = now_ms();
    double hp_t = t_start;   // YK_PROFILE_HOST: where the host time of the cycle goes (printed by yk_destroy)
    auto hp = [&](int k) { if (e->hp_on) { const double t = now_ms(); e->hp[k] += t - hp_t; hp_t = t; } };
    // the orderer's per-cycle setup (host only) runs on the helper thread while this thread uploads stale tables and
    // starts the initial node order on the device
    std::vector<uint32_t>& pending = e->pending;
    double begin_ms = 0;
    bool gang_too_big = false;
    setup_commit_tables(e);
    // device commit: forced (every eligible cycle), or automatic (cycles whose asks come in long uniform runs: yk_uniform.h);
    // binpacking cycles only under YK_FLAG_BINPACKING_DEVICE, and never on the round commit
    const bool bp = e->cfg.policy == YK_POLICY_BINPACKING;
    const bool dev_policy = e->cfg.policy == YK_POLICY_FAIR || (bp && e->bp_device);
    const bool force_lattice = e->lt_allowed && e->lt_force && dev_policy;
    const bool auto_lattice = e->lt_allowed && !e->lt_force && e->lt_auto && e->un_min > 0 && dev_policy;
    yklt::Scan scan;   // the pending scan's hints for the commit choice
    // a speculative round-commit launch reads the ask states as the cycle began: copied before the pending scan rewrites them
    const bool spec = spec_gate(e, max_bindings, auto_lattice);
    if (spec) memcpy(e->h_sp_state.p, e->a_state.data(), e->a_hi);
    e->sp_live = e->sp_adopt = false;
    e->worker.submit([&] {
        const double t_b = now_ms();
        pending.clear();
        pending.reserve(e->a_hi);
        bool any_gang = false;
        const bool hints = auto_lattice && !spec;   // (a speculative cycle's calling thread takes them: below)
        if (hints) for (uint32_t n = 0; n < e->n_hi; ++n) if (e->n_present[n]) scan.taints |= e->n_taint[n];
        for (uint32_t a = 0; a < e->a_hi; ++a) {
            uint8_t& st = e->a_state[a];
            if (st == yk::ST_ABSENT || st == yk::ST_ALLOCATED) continue;
            st = yk::ST_PENDING;   // failed / skipped asks are tried again every cycle, like the reference
            if (!e->p_present[e->a_app[a]]) continue;
            pending.push_back(a);
            any_gang = any_gang || e->a_gang[a] != YK_NONE;
            if (hints) scan.add(e->cm.t, e->a_sigid.data(), a);
        }
        e->cycle_has_gang = any_gang;
        if (!spec) e->rd_taints = scan.taints;
        if (any_gang) {   // a gang that no batch can hold is an argument error: found before anything is committed
            std::unordered_map<uint64_t, uint32_t> members;
            for (uint32_t a : pending)
                if (e->a_gang[a] != YK_NONE && ++members[((uint64_t)e->a_app[a] << 32) | e->a_gang[a]] > e->batch) gang_too_big = true;
        }
        yk::Tables& t = e->ord.t;
        t.D = e->D; t.maxA = e->maxA; t.maxP = e->maxP; t.nq = e->nq;
        t.a_req = e->a_req.p; t.a_prio = e->a_prio.data(); t.a_create = e->a_create.data(); t.a_app = e->a_app.data();
        t.a_flags = e->a_flags.data(); t.a_cause = e->a_cause.data(); t.a_gang = e->a_gang.data(); t.a_state = e->a_state.data();
        t.p_queue = e->p_queue.data(); t.p_submit = e->p_submit.data(); t.p_present = e->p_present.data();
        t.q_parent = e->q_parent.data(); t.q_guar = e->q_guar.data(); t.q_max = e->q_max.data(); t.q_alloc = e->q_alloc.data(); t.p_alloc = e->p_alloc.data();
        t.q_sort = e->q_sort.data();
        t.q_prio_offset = e->q_prio_offset.data(); t.q_prio_fence = e->q_prio_fence.data();
        t.p_user = e->p_user.data(); t.n_ul = e->n_ul; t.ul_queue = e->ul_queue.data(); t.ul_user = e->ul_user.data();
        t.ul_max = e->ul_max.data(); t.ul_alloc = e->ul_alloc.data();
        if (!gang_too_big) e->ord.begin_cycle(pending);
        if (!gang_too_big && !spec) epoch_rows(e, pending);
        if (!gang_too_big && !spec) scan.done(e->cm.t, pending, force_lattice, e->a_shape);
        e->ep_uploaded = false; e->ep_landed = true;
        begin_ms = now_ms() - t_b;
    });
    hp(0);
    int rc = upload_tables(e);
    // the device scores and sorts the nodes while the helper thread still sets the orderer up
    e->order_enqueued = false;
    if (!rc) { rc = device_order(e); e->order_enqueued = rc == YK_OK && e->nlive > 0; }
    // ... and, where the cycle may be a round-commit one, orders the asks and starts the round kernel on them
    if (!rc && spec) rc = spec_launch(e, max_bindings);
    // ... and takes over the pending scan's commit-choice hints and the epoch rows, which read only which asks the scan keeps
    // (the states as the cycle began, the present applications): they run next to the helper's orderer set-up, not after it
    if (spec) {
        std::vector<uint32_t>& kept = e->sp_pending;
        kept.clear();
        for (uint32_t n = 0; n < e->n_hi; ++n) if (e->n_present[n]) scan.taints |= e->n_taint[n];
        for (uint32_t a = 0; a < e->a_hi; ++a) {
            const uint8_t st = e->h_sp_state[a];
            if (st == yk::ST_ABSENT || st == yk::ST_ALLOCATED || !e->p_present[e->a_app[a]]) continue;
            kept.push_back(a);
            scan.add(e->cm.t, e->a_sigid.data(), a);
        }
        e->rd_taints = scan.taints;
        epoch_rows(e, kept);
    }
    const double t_a = now_ms();
    hp(1);
    e->worker.wait();
    hp(2);
    e->st.host_ms[0] += t_a - t_start;
    e->st.host_ms[1] += begin_ms;
    if (spec && !gang_too_big) scan.done(e->cm.t, pending, force_lattice, e->a_shape);
    if (rc || gang_too_big) {
        const int rcd = spec_discard(e);
        if (rc) return rc;
        return rcd ? rcd : e->fail(YK_ERR_ARG, yk::GANG_TOO_BIG);
    }

    Cycle c;
    c.max_bindings = max_bindings; c.out = out;
    // which commit the cycle starts on, and its first batch (a hand-off refills the slot, still unlaunched)
    Slot& first = e->slot[0];
    first.B = 0; first.nchunks = 0;
    const yklt::ChoiceIn in{e->ord, e->cm.t, pending, e->n_hi, e->n_present.data(), e->n_total.p, e->maxN, e->n_rank.data(),
                            &e->ranks_unique, &e->cycle_has_gang, force_lattice, auto_lattice, e->bp_device, e->un_min, e->rd_min,
                            scan, e->batch, e->maxA, max_bindings, e->a_shape.data(), e->a_sigid.data(), first.asks, first.snap,
                            e->h_lt_meta.p, e->h_lt_shp.p, e->h_lt_sig.p, e->un_segs, e->st};
    yklt::Choice choice;
    if (!yklt::choose_commit(in, choice)) rc = e->fail(YK_ERR_ARG, yk::GANG_TOO_BIG);
    e->lt_active = false;
    hp(3);
    {
        const int rcv = rc ? spec_discard(e) : spec_verify(e, choice);
        if (!rc) rc = rcv;
    }
    hp(8);
    if (!rc) {
        if (choice.device) {
            e->lt_active = true;
            e->order_enqueued = false;   // consumed by lt_prepare; a hand-over sorts again from the exported tables
            e->st.lattice_cycles++;
            bool handoff = false;
            rc = run_lattice(e, c, choice, handoff);
            if (!rc) {
                const int rce = lt_export(e);   // node tables current again, host and device
                e->lt_active = false;
                rc = rce;
            }
            if (!rc) {
                const int* h = e->h_lt_hdr.p;
                e->lt_total_subruns += (uint64_t)h[yklt::H_SUBRUNS];
                e->st.lattice_subruns += (uint64_t)h[yklt::H_SUBRUNS]; e->st.lattice_fullscans += (uint64_t)h[yklt::H_FULLSCANS];
                e->st.lattice_sorts += (uint64_t)h[yklt::H_SORTS]; e->st.lattice_elements += (uint64_t)h[yklt::H_ELEMS];
                e->st.lattice_quick += (uint64_t)h[yklt::H_QUICK];
            }
            if (!rc && handoff && c.n < max_bindings) {
                size_t b = e->batch;
                rc = yk::fill_batch(e->ord, b, e->batch, (size_t)max_bindings - c.n, first.asks, first.snap, e->st)
                         ? run_host(e, c) : e->fail(YK_ERR_ARG, yk::GANG_TOO_BIG);
            }
        } else {
            rc = run_host(e, c);
        }
    }
    hp(4);
    e->sp_adopt = false;
    // ---- always: leave host and device node tables current, persist what was bound, no ask left in flight ----
    int rc_end = YK_OK;
    if (e->lt_active) { rc_end = lt_export(e); e->lt_active = false; }
    else rc_end = end_epoch(e, false);
    e->cm.begin_epoch(e->epochW);   // nothing touched any more
    for (int k = 0; k < 4; ++k) { e->st.dbg[k] += e->cm.dbg[k]; e->cm.dbg[k] = 0; }
    for (int k = 0; k < 6; ++k) { e->st.prof[k] += e->cm.prof[k]; e->cm.prof[k] = 0; }
    if (cudaStreamSynchronize(e->stream) != cudaSuccess && !rc && !rc_end) rc_end = e->fail(YK_ERR_CUDA, "cudaStreamSynchronize at the end of the cycle");
    hp(5);
    if (rc) {
        // the cycle broke off: the bindings made so far stand (they are returned), every ask still in flight is pending
        // again, and the queue / application accounting is rebuilt from exactly the bindings returned
        e->worker.wait();
        for (Slot& sl : e->slot) { if (sl.B > 0 && sl.nchunks > 0) cudaEventSynchronize(sl.ev[(size_t)sl.nchunks - 1]); sl.asks.clear(); sl.B = 0; sl.nchunks = 0; }
        for (uint32_t a : pending) if (e->a_state[a] == yk::ST_TENTATIVE) e->a_state[a] = yk::ST_PENDING;
        for (uint32_t i = 0; i < c.n; ++i) {   // (the commit has already taken them from their nodes)
            int64_t r[8];
            ask_request(e, out[i].ask, r);
            alloc_move(e, out[i].ask, r, false);
        }
    } else {
        e->ord.finish();
    }
    for (uint32_t a : e->ord.slow_list) {
        if (slow && n_slow && *n_slow < slow_cap) slow[(*n_slow)++] = a;
    }
    for (uint32_t a : pending) if (e->a_state[a] == yk::ST_SKIPPED) e->st.skipped++;
    *n_out = c.n;
    e->st.cycles++;
    hp(6);
    e->hp_n++;
    e->st.total_ms += now_ms() - t_start;
    return rc ? rc : rc_end;
}

namespace {

constexpr uint32_t FILTER_CHUNK = 4096;      // asks per yk_filter_kernel launch at most
constexpr size_t FILTER_WORDS = 1u << 24;    // device words per chunk at most (bitmap + tile counts + counts + window)
constexpr int FILTER_AC = 32;                // asks per shared-memory stage of yk_filter_kernel
constexpr uint32_t PN_ROWS = 4096;           // victim lists per yk_preemption_nodes chunk at most
constexpr uint32_t PN_ENTRIES = 1u << 18;    // victim entries per chunk at most, unless one list alone is longer
constexpr size_t PN_WORDS = 1u << 24;        // read-back words per chunk at most ([lists][2k + 3])

void launch_filter(int D, const YkFilterArgs& a, dim3 grid, cudaStream_t s) {
    switch (D) {
        case 1: yk_filter_kernel<1, FILTER_AC><<<grid, YK_FILTER_THREADS, 0, s>>>(a); break;
        case 2: yk_filter_kernel<2, FILTER_AC><<<grid, YK_FILTER_THREADS, 0, s>>>(a); break;
        case 3: yk_filter_kernel<3, FILTER_AC><<<grid, YK_FILTER_THREADS, 0, s>>>(a); break;
        case 4: yk_filter_kernel<4, FILTER_AC><<<grid, YK_FILTER_THREADS, 0, s>>>(a); break;
        case 5: yk_filter_kernel<5, FILTER_AC><<<grid, YK_FILTER_THREADS, 0, s>>>(a); break;
        case 6: yk_filter_kernel<6, FILTER_AC><<<grid, YK_FILTER_THREADS, 0, s>>>(a); break;
        case 7: yk_filter_kernel<7, FILTER_AC><<<grid, YK_FILTER_THREADS, 0, s>>>(a); break;
        default: yk_filter_kernel<8, FILTER_AC><<<grid, YK_FILTER_THREADS, 0, s>>>(a); break;
    }
}

template <typename T>
cudaError_t grow(Dev<T>& d, size_t n) { return d.n < n ? d.alloc(n) : cudaSuccess; }
template <typename T>
cudaError_t grow(Pin<T>& h, size_t n) { return h.n < n ? h.alloc(n) : cudaSuccess; }

// Enqueue every present node's sort key under (policy, w) into f_key_in / f_val_in[0, nlive) (NodeID-rank order), with the NaN
// flag copied to h_f_flag (valid after the stream's next synchronise).  The buffers are the filter's own, so a cycle's sort
// buffers are never touched.  Needs e->nlive > 0 and the tables uploaded.
int filter_keys(yk_engine* e, uint32_t policy, const YkWeights& w) {
    cudaStream_t s = e->stream;
    const size_t N = e->maxN;
    const uint32_t nlive = e->nlive;
    if (e->f_key_in.n < N) {
        CK(e->f_key_in.alloc(N)); CK(e->f_key_out.alloc(N)); CK(e->f_val_in.alloc(N)); CK(e->f_val_out.alloc(N));
        size_t tb = 0;
        CK(cub::DeviceRadixSort::SortPairs(nullptr, tb, e->f_key_in.p, e->f_key_out.p, e->f_val_in.p, e->f_val_out.p, (int)N, 0, 64, s));
        e->f_cub_bytes = tb;
        CK(e->f_cub.alloc(tb));
        CK(e->f_flag.alloc(1)); CK(e->h_f_flag.alloc(1));
    }
    CK(cudaMemsetAsync(e->f_flag.p, 0, sizeof(int), s));
    yk_key_kernel<<<(nlive + 255) / 256, 256, 0, s>>>(e->D, policy, w, e->d_total.p, e->d_avail.p, e->maxN, e->d_by_rank.p,
                                                      (int)nlive, e->f_key_in.p, e->f_val_in.p, e->f_flag.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(e->h_f_flag.p, e->f_flag.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    e->st.other_launches += 1;
    e->st.d2h_bytes += 4;
    return YK_OK;
}

// Enqueue the node order under (policy, w) at this moment (ascending (score, NodeID rank, index)) into f_val_out[0, nlive), with
// the NaN flag as filter_keys leaves it.  yk_filter_nodes and yk_preemption_nodes use it with the engine's current setting.
int filter_order(yk_engine* e, uint32_t policy, const YkWeights& w) {
    const int rc = filter_keys(e, policy, w);
    if (rc) return rc;
    size_t tb = e->f_cub_bytes;
    CK(cub::DeviceRadixSort::SortPairs(e->f_cub.p, tb, e->f_key_in.p, e->f_key_out.p, e->f_val_in.p, e->f_val_out.p, (int)e->nlive, 0, 64,
                                       e->stream));
    e->st.other_launches += 10;   // cub radix sort (histogram, exclusive sum, 8 onesweep passes), as device_order
    return YK_OK;
}

}  // namespace

extern "C" {

int yk_ask_states(yk_engine* e, uint32_t n, const uint32_t* idx, uint8_t* out) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!idx || !out)) return e->fail(YK_ERR_ARG, "yk_ask_states: null array");
    for (uint32_t i = 0; i < n; ++i) {
        if (idx[i] >= e->maxA) return e->fail(YK_ERR_ARG, "yk_ask_states: index beyond max_asks");
        out[i] = e->a_state[idx[i]];
    }
    return YK_OK;
}

int yk_nodes_available(yk_engine* e, uint32_t n, const uint32_t* idx, int64_t* out) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!idx || !out)) return e->fail(YK_ERR_ARG, "yk_nodes_available: null array");
    for (uint32_t i = 0; i < n; ++i) {
        if (idx[i] >= e->maxN) return e->fail(YK_ERR_ARG, "yk_nodes_available: index beyond max_nodes");
        for (int k = 0; k < e->D; ++k) out[(size_t)k * n + i] = e->n_avail[(size_t)k * e->maxN + idx[i]];
    }
    return YK_OK;
}

static int evaluate_phase(yk_engine* e, uint32_t ask, uint32_t node, int allocate) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (ask >= e->maxA || node >= e->maxN) return e->fail(YK_ERR_ARG, "yk_evaluate: index out of range");
    if (e->a_state[ask] == yk::ST_ABSENT || !e->n_present[node]) return YK_FAIL_ABSENT;
    int rc = upload_tables(e);
    if (rc) return rc;
    yk_evaluate_kernel<<<1, 32, 0, e->stream>>>(e->D, e->d_total.p, e->d_avail.p, e->maxN, e->d_taint.p, e->d_label.p,
                                                e->d_flags.p, e->d_areq.p, e->d_atol.p, e->d_aneed.p, e->d_adeny.p,
                                                e->d_anode.p, e->maxA, ask, node, allocate, e->d_flag.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(e->h_flag.p, e->d_flag.p, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->st.other_launches++;
    return e->h_flag[0];
}

int yk_evaluate(yk_engine* e, uint32_t ask, uint32_t node) { return evaluate_phase(e, ask, node, 1); }
int yk_evaluate_reserve(yk_engine* e, uint32_t ask, uint32_t node) { return evaluate_phase(e, ask, node, 0); }

int yk_node_scores(yk_engine* e, uint32_t n, const uint32_t* idx, double* out) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!idx || !out)) return e->fail(YK_ERR_ARG, "yk_node_scores: null array");
    if (n > e->maxN) return e->fail(YK_ERR_ARG, "yk_node_scores: more indices than max_nodes");
    for (uint32_t i = 0; i < n; ++i) if (idx[i] >= e->maxN) return e->fail(YK_ERR_ARG, "yk_node_scores: index beyond max_nodes");
    if (!n) return YK_OK;
    int rc = upload_tables(e);
    if (rc) return rc;
    memcpy(e->h_snode.p, idx, 4 * (size_t)n);
    CK(cudaMemcpyAsync(e->d_val_in.p, e->h_snode.p, 4 * (size_t)n, cudaMemcpyHostToDevice, e->stream));
    yk_score_kernel<<<(n + 255) / 256, 256, 0, e->stream>>>(e->D, e->cfg.policy, e->w, e->d_total.p, e->d_avail.p, e->maxN,
                                                           e->d_val_in.p, (int)n, e->d_scores.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(e->h_scores.p, e->d_scores.p, 8 * (size_t)n, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    memcpy(out, e->h_scores.p, 8 * (size_t)n);
    e->st.other_launches++;
    return YK_OK;
}

// Every reader of the setting (the cycle's set-up, commit choice and launches, the queries above) reads e->cfg.policy / e->w
// when it runs, and the device state kept between cycles (the lattice records and order, the uniform runs' re-keyed order) is
// rebuilt from the cycle's own initial order: replacing the two here is all a switch needs.
int yk_node_sort_set(yk_engine* e, uint32_t policy, const double* weights) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (!weights) return e->fail(YK_ERR_ARG, "yk_node_sort_set: null weights");
    if (policy != YK_POLICY_FAIR && policy != YK_POLICY_BINPACKING) return e->fail(YK_ERR_ARG, "yk_node_sort_set: unknown node sort policy");
    YkWeights w{};
    for (int k = 0; k < e->D; ++k) {
        if (!std::isfinite(weights[k])) return e->fail(YK_ERR_ARG, "yk_node_sort_set: NaN or infinite weight");
        w.w[k] = weights[k];
    }
    int rc = upload_tables(e);
    if (rc) return rc;
    if (e->nlive) {   // all or nothing: every present node is scored under the new setting by the cycle's own key kernel first
        rc = filter_keys(e, policy, w);
        if (rc) return rc;
        CK(cudaStreamSynchronize(e->stream));
        if (e->h_f_flag[0]) return e->fail(YK_ERR_RANGE, "yk_node_sort_set: a present node scores NaN under the new setting (zero total "
                                                         "on a weighted resource); the old setting is kept");
    }
    e->cfg.policy = policy;
    for (int k = 0; k < 8; ++k) e->cfg.weights[k] = w.w[k];
    e->w = w;
    return YK_OK;
}

int yk_preemption_search(yk_engine* e, uint32_t nq, const uint32_t* ask, const uint32_t* node, const uint32_t* voff,
                         const int64_t* vreq, const uint32_t* start, int32_t* out) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (nq && (!ask || !node || !voff || !start || !out)) return e->fail(YK_ERR_ARG, "yk_preemption_search: null array");
    if (!nq) return YK_OK;
    const uint32_t nv = voff[nq];
    if (nv && !vreq) return e->fail(YK_ERR_ARG, "yk_preemption_search: null victim_req");
    for (uint32_t i = 0; i < nq; ++i) {
        if (ask[i] >= e->maxA || node[i] >= e->maxN || e->a_state[ask[i]] == yk::ST_ABSENT || !e->n_present[node[i]])
            return e->fail(YK_ERR_ARG, "yk_preemption_search: unknown ask or node");
        if (voff[i] > voff[i + 1]) return e->fail(YK_ERR_ARG, "yk_preemption_search: victim_off must be non-decreasing");
    }
    int rc = upload_tables(e);
    if (rc) return rc;
    const int D = e->D;
    // device buffers are kept between calls and only grow (a cudaMalloc per call costs more than the search)
    Dev<uint32_t>& d_q = e->pre_q; Dev<int64_t>& d_v = e->pre_v; Dev<int32_t>& d_o = e->pre_o;
    if (d_q.n < (size_t)nq * 4 + 1) CK(d_q.alloc(((size_t)nq * 4 + 1) * 2));
    if (d_v.n < (size_t)std::max<uint32_t>(nv, 1) * D) CK(d_v.alloc((size_t)std::max<uint32_t>(nv, 1) * D * 2));
    if (d_o.n < nq) CK(d_o.alloc((size_t)nq * 2));
    cudaStream_t s = e->stream;
    CK(cudaMemcpyAsync(d_q.p, ask, 4 * (size_t)nq, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_q.p + nq, node, 4 * (size_t)nq, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_q.p + 2 * (size_t)nq, voff, 4 * ((size_t)nq + 1), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_q.p + 3 * (size_t)nq + 1, start, 4 * (size_t)nq, cudaMemcpyHostToDevice, s));
    if (nv) CK(cudaMemcpyAsync(d_v.p, vreq, 8 * (size_t)nv * D, cudaMemcpyHostToDevice, s));
    const int threads = 128, warps_per_block = threads / 32;
    yk_preempt_kernel<<<(nq + warps_per_block - 1) / warps_per_block, threads, 0, s>>>(
        D, e->d_total.p, e->d_avail.p, e->maxN, e->d_taint.p, e->d_label.p, e->d_flags.p, e->d_areq.p, e->d_atol.p,
        e->d_aneed.p, e->d_adeny.p, e->d_anode.p, e->maxA, (int)nq, d_q.p, d_q.p + nq, d_q.p + 2 * (size_t)nq, d_v.p,
        std::max<uint32_t>(nv, 1), d_q.p + 3 * (size_t)nq + 1, d_o.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, d_o.p, 4 * (size_t)nq, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    e->st.other_launches++;
    return YK_OK;
}

int yk_filter_nodes(yk_engine* e, uint32_t n, const uint32_t* asks, int allocate, uint32_t skip, uint32_t k,
                    uint32_t* nodes_out, uint32_t* n_pass, uint32_t* counts) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && !asks) return e->fail(YK_ERR_ARG, "yk_filter_nodes: null asks");
    if (k && !nodes_out) return e->fail(YK_ERR_ARG, "yk_filter_nodes: null nodes_out with k > 0");
    for (uint32_t i = 0; i < n; ++i) if (asks[i] >= e->maxA) return e->fail(YK_ERR_ARG, "yk_filter_nodes: ask index beyond max_asks");
    if (!n) return YK_OK;
    int rc = upload_tables(e);
    if (rc) return rc;
    const uint32_t nlive = e->nlive;
    if (nlive == 0) {   // no node: nothing passes, nothing to count
        if (k) std::fill(nodes_out, nodes_out + (size_t)n * k, YK_NONE);
        if (n_pass) std::fill(n_pass, n_pass + n, 0u);
        if (counts) std::fill(counts, counts + (size_t)n * YK_FILTER_SLOTS, 0u);
        return YK_OK;
    }
    static_assert(YK_FILTER_SLOTS == YK_FILTER_NSLOT && YK_FILTER_RESERVED == YK_FILTER_RES && YK_FAIL_ABSENT == YK_FILTER_ABSENT,
                  "slot numbers of ykgpu.h and yk_filter.cuh");
    const int D = e->D;
    cudaStream_t s = e->stream;
    const int tiles = (int)((nlive + YK_FILTER_THREADS - 1) / YK_FILTER_THREADS), W = tiles * YK_FILTER_TW;
    const size_t row_words = (size_t)W + tiles + YK_FILTER_SLOTS + k;
    const uint32_t chunk = (uint32_t)std::min<size_t>({(size_t)n, FILTER_CHUNK, std::max<size_t>(1, FILTER_WORDS / row_words)});
    // device buffers are kept between calls and only grow
    CK(grow(e->f_asks, chunk)); CK(grow(e->h_f_asks, chunk));
    CK(grow(e->f_bits, (size_t)chunk * W)); CK(grow(e->f_tcnt, (size_t)chunk * tiles));
    CK(grow(e->f_counts, (size_t)chunk * YK_FILTER_SLOTS)); CK(grow(e->h_f_counts, (size_t)chunk * YK_FILTER_SLOTS));
    if (k) { CK(grow(e->f_out, (size_t)chunk * k)); CK(grow(e->h_f_out, (size_t)chunk * k)); }
    rc = filter_order(e, e->cfg.policy, e->w);
    if (rc) return rc;

    YkFilterArgs a{};
    a.total = e->d_total.p; a.avail = e->d_avail.p; a.ldn = e->maxN;
    a.taint = e->d_taint.p; a.label = e->d_label.p; a.flags = e->d_flags.p;
    a.sorted = e->f_val_out.p; a.nlive = (int)nlive;
    a.a_req = e->d_areq.p; a.a_tol = e->d_atol.p; a.a_need = e->d_aneed.p; a.a_deny = e->d_adeny.p; a.a_node = e->d_anode.p;
    a.lda = e->maxA;
    a.asks = e->f_asks.p; a.allocate = allocate ? 1 : 0;
    a.bits = e->f_bits.p; a.tilecnt = e->f_tcnt.p; a.counts = e->f_counts.p;
    a.W = W; a.tiles = tiles;
    for (uint32_t c0 = 0; c0 < n; c0 += chunk) {
        const uint32_t rows = std::min(chunk, n - c0);
        for (uint32_t i = 0; i < rows; ++i) {   // an ask that is not present is sent as YK_NONE: every node counts as YK_FAIL_ABSENT
            const uint32_t x = asks[c0 + i];
            e->h_f_asks[i] = e->a_state[x] == yk::ST_ABSENT ? YK_NONE : x;
        }
        CK(cudaMemcpyAsync(e->f_asks.p, e->h_f_asks.p, 4 * (size_t)rows, cudaMemcpyHostToDevice, s));
        CK(cudaMemsetAsync(e->f_counts.p, 0, 4 * (size_t)rows * YK_FILTER_SLOTS, s));
        // grid.y sized so that tiles x splits fills the device's resident CTA slots about once
        const int splits = std::max(1, std::min<int>((int)rows, e->slots / tiles));
        a.rows = (int)rows;
        a.per = (int)((rows + splits - 1) / splits);
        launch_filter(D, a, dim3((unsigned)tiles, (unsigned)((rows + a.per - 1) / a.per)), s);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(e->h_f_counts.p, e->f_counts.p, 4 * (size_t)rows * YK_FILTER_SLOTS, cudaMemcpyDeviceToHost, s));
        e->st.other_launches += 1;
        e->st.h2d_bytes += 4 * (size_t)rows;
        e->st.d2h_bytes += 4 * (size_t)rows * YK_FILTER_SLOTS;
        if (k) {
            yk_filter_compact_kernel<<<(rows + 3) / 4, 128, 0, s>>>(e->f_bits.p, e->f_tcnt.p, e->f_counts.p, e->f_val_out.p, (int)rows,
                                                                    W, tiles, skip, k, e->f_out.p);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(e->h_f_out.p, e->f_out.p, 4 * (size_t)rows * k, cudaMemcpyDeviceToHost, s));
            e->st.other_launches += 1;
            e->st.d2h_bytes += 4 * (size_t)rows * k;
        }
        CK(cudaStreamSynchronize(s));
        if (e->h_f_flag[0]) return e->fail(YK_ERR_RANGE, "yk_filter_nodes: NaN node score (zero total on a weighted resource)");
        if (k) memcpy(nodes_out + (size_t)c0 * k, e->h_f_out.p, 4 * (size_t)rows * k);
        if (counts) memcpy(counts + (size_t)c0 * YK_FILTER_SLOTS, e->h_f_counts.p, 4 * (size_t)rows * YK_FILTER_SLOTS);
        if (n_pass) for (uint32_t i = 0; i < rows; ++i) n_pass[c0 + i] = e->h_f_counts[(size_t)i * YK_FILTER_SLOTS];
    }
    return YK_OK;
}

int yk_preemption_nodes(yk_engine* e, uint32_t n, const uint32_t* asks, const uint32_t* victim_off, const uint32_t* victims,
                        uint32_t skip, uint32_t k, uint32_t* nodes_out, uint32_t* need_out, uint32_t* n_fit,
                        uint32_t* best_node, uint32_t* best_need) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!asks || !victim_off)) return e->fail(YK_ERR_ARG, "yk_preemption_nodes: null asks or victim_off");
    if (k && !nodes_out) return e->fail(YK_ERR_ARG, "yk_preemption_nodes: null nodes_out with k > 0");
    if (!n) return YK_OK;
    if (victim_off[0] != 0) return e->fail(YK_ERR_ARG, "yk_preemption_nodes: victim_off[0] must be 0");
    for (uint32_t i = 0; i < n; ++i) {
        if (asks[i] >= e->maxA) return e->fail(YK_ERR_ARG, "yk_preemption_nodes: ask index beyond max_asks");
        if (victim_off[i] > victim_off[i + 1]) return e->fail(YK_ERR_ARG, "yk_preemption_nodes: victim_off must be non-decreasing");
    }
    const uint32_t nv = victim_off[n];
    if (nv && !victims) return e->fail(YK_ERR_ARG, "yk_preemption_nodes: null victims");
    if (e->pn_seen.size() < e->maxA) { e->pn_seen.assign(e->maxA, 0); e->pn_stamp = 0; }
    for (uint32_t i = 0; i < n; ++i) {
        if (++e->pn_stamp == 0) { std::fill(e->pn_seen.begin(), e->pn_seen.end(), 0u); e->pn_stamp = 1; }
        for (uint32_t j = victim_off[i]; j < victim_off[i + 1]; ++j) {
            const uint32_t v = victims[j];
            if (v >= e->maxA) return e->fail(YK_ERR_ARG, "yk_preemption_nodes: victim index beyond max_asks");
            if (e->pn_seen[v] == e->pn_stamp) return e->fail(YK_ERR_ARG, "yk_preemption_nodes: the same victim twice in one list");
            e->pn_seen[v] = e->pn_stamp;
        }
    }
    for (uint32_t j = 0; j < nv; ++j)
        if (e->a_state[victims[j]] != yk::ST_ALLOCATED) return e->fail(YK_ERR_STATE, "yk_preemption_nodes: a victim holds no allocation");
    int rc = upload_tables(e);
    if (rc) return rc;
    const uint32_t nlive = e->nlive;
    auto write_empty = [&](uint32_t i0, uint32_t i1) {   // asks i0 .. i1-1 have no fitting node
        if (k) std::fill(nodes_out + (size_t)i0 * k, nodes_out + (size_t)i1 * k, YK_NONE);
        if (k && need_out) std::fill(need_out + (size_t)i0 * k, need_out + (size_t)i1 * k, 0u);
        if (n_fit) std::fill(n_fit + i0, n_fit + i1, 0u);
        if (best_node) std::fill(best_node + i0, best_node + i1, YK_NONE);
        if (best_need) std::fill(best_need + i0, best_need + i1, 0u);
    };
    if (nlive == 0) { write_empty(0, n); return YK_OK; }   // no node: no victim is on a present node

    const int D = e->D;
    cudaStream_t s = e->stream;
    CK(grow(e->pn_pos, e->maxN));
    rc = filter_order(e, e->cfg.policy, e->w);
    if (rc) return rc;
    yk_pn_pos_kernel<<<(nlive + 255) / 256, 256, 0, s>>>(e->f_val_out.p, (int)nlive, e->pn_pos.p);
    CK(cudaGetLastError());
    e->st.other_launches += 1;
    const auto bits = [](uint32_t x) { return x ? 32 - __builtin_clz(x) : 0; };
    const int pbits = std::max(1, bits(nlive - 1));
    const size_t row_words = 2 * (size_t)k + 3;
    const uint32_t rows_cap = (uint32_t)std::min<size_t>(PN_ROWS, std::max<size_t>(1, PN_WORDS / row_words));
    for (uint32_t c0 = 0; c0 < n;) {
        // a chunk is whole lists: it ends before the list that would take it past PN_ENTRIES entries or rows_cap lists (a
        // longer list is a chunk of its own)
        uint32_t c1 = c0 + 1;
        while (c1 < n && c1 - c0 < rows_cap && victim_off[c1 + 1] - victim_off[c0] <= PN_ENTRIES) ++c1;
        const uint32_t rows = c1 - c0, raw = victim_off[c1] - victim_off[c0];
        const size_t head_words = 2 * (size_t)rows + 1;
        CK(grow(e->h_pn_in, head_words + 2 * (size_t)raw));
        uint32_t* h_asks = e->h_pn_in.p;
        uint32_t* h_off = h_asks + rows;
        uint32_t* h_vic = h_off + rows + 1;
        uint32_t* h_node = h_vic + raw;
        uint32_t m = 0;   // entries kept: victims bound to a present node, of asks that are present
        for (uint32_t r = 0; r < rows; ++r) {
            const uint32_t i = c0 + r;
            h_asks[r] = asks[i];
            h_off[r] = m;
            if (e->a_state[asks[i]] == yk::ST_ABSENT) continue;
            for (uint32_t j = victim_off[i]; j < victim_off[i + 1]; ++j) {
                const uint32_t v = victims[j], node = e->a_bound[v];
                if (node >= e->maxN || !e->n_present[node]) continue;
                h_vic[m] = v; h_node[m] = node; ++m;
            }
        }
        h_off[rows] = m;
        if (m) {
            const int end_bit = pbits + std::max(1, bits(rows - 1));
            CK(grow(e->pn_in, head_words + 2 * (size_t)raw));
            CK(grow(e->pn_key_in, m)); CK(grow(e->pn_key_out, m)); CK(grow(e->pn_val_in, m)); CK(grow(e->pn_val_out, m));
            CK(grow(e->pn_head, m)); CK(grow(e->pn_incl, m)); CK(grow(e->pn_gask, m)); CK(grow(e->pn_gnode, m));
            CK(grow(e->pn_goff, (size_t)m + 1)); CK(grow(e->pn_start, m)); CK(grow(e->pn_res, m)); CK(grow(e->pn_vreq, (size_t)D * m));
            CK(grow(e->pn_out, rows * row_words)); CK(grow(e->h_pn_out, rows * row_words));
            size_t sort_b = 0, scan_b = 0;
            CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_b, e->pn_key_in.p, e->pn_key_out.p, e->pn_val_in.p, e->pn_val_out.p,
                                               (int)m, 0, end_bit, s));
            CK(cub::DeviceScan::InclusiveSum(nullptr, scan_b, e->pn_head.p, e->pn_incl.p, (int)m, s));
            CK(grow(e->pn_cub, std::max(sort_b, scan_b)));
            uint32_t* d_asks = e->pn_in.p;
            uint32_t* d_off = d_asks + rows;
            uint32_t* d_vic = d_off + rows + 1;
            uint32_t* d_node = d_vic + raw;
            CK(cudaMemcpyAsync(d_asks, h_asks, 4 * (head_words + m), cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(d_node, h_node, 4 * (size_t)m, cudaMemcpyHostToDevice, s));
            const unsigned blocks = (m + 255) / 256;
            yk_pn_key_kernel<<<blocks, 256, 0, s>>>(d_off, (int)rows, d_node, e->pn_pos.p, (int)m, pbits, e->pn_key_in.p,
                                                    e->pn_val_in.p);
            size_t tb = sort_b;   // stable: the entries of one (list, node) group stay in list order
            CK(cub::DeviceRadixSort::SortPairs(e->pn_cub.p, tb, e->pn_key_in.p, e->pn_key_out.p, e->pn_val_in.p, e->pn_val_out.p,
                                               (int)m, 0, end_bit, s));
            yk_pn_head_kernel<<<blocks, 256, 0, s>>>(e->pn_key_out.p, (int)m, e->pn_head.p);
            tb = scan_b;
            CK(cub::DeviceScan::InclusiveSum(e->pn_cub.p, tb, e->pn_head.p, e->pn_incl.p, (int)m, s));
            yk_pn_group_kernel<<<blocks, 256, 0, s>>>(D, e->pn_key_out.p, e->pn_val_out.p, e->pn_incl.p, (int)m, pbits, d_asks, d_vic,
                                                      e->f_val_out.p, e->d_areq.p, e->maxA, e->pn_gask.p, e->pn_gnode.p,
                                                      e->pn_goff.p, e->pn_vreq.p);
            CK(cudaMemsetAsync(e->pn_start.p, 0, 4 * (size_t)m, s));
            // every (list, node) group is one query of the single-query search, start 0: the answers are yk_preemption_search's
            yk_preempt_kernel<<<(m + 3) / 4, 128, 0, s>>>(
                D, e->d_total.p, e->d_avail.p, e->maxN, e->d_taint.p, e->d_label.p, e->d_flags.p, e->d_areq.p, e->d_atol.p,
                e->d_aneed.p, e->d_adeny.p, e->d_anode.p, e->maxA, (int)m, e->pn_gask.p, e->pn_gnode.p, e->pn_goff.p, e->pn_vreq.p,
                m, e->pn_start.p, e->pn_res.p);
            yk_pn_rank_kernel<<<(rows + 3) / 4, 128, 0, s>>>(d_off, e->pn_incl.p, e->pn_res.p, e->pn_gnode.p, (int)rows, skip, k,
                                                             e->pn_out.p);
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(e->h_pn_out.p, e->pn_out.p, 4 * rows * row_words, cudaMemcpyDeviceToHost, s));
            // 5 kernels of yk_preempt_nodes.cuh / yk_kernels.cuh, the cub radix sort (histogram, exclusive sum, one onesweep
            // pass per 8 key bits) and the cub scan (init, scan)
            e->st.other_launches += 5 + 2 + (end_bit + 7) / 8 + 2;
            e->st.h2d_bytes += 4 * (head_words + 2 * (size_t)m);
            e->st.d2h_bytes += 4 * rows * row_words;
        }
        CK(cudaStreamSynchronize(s));
        if (e->h_f_flag[0]) return e->fail(YK_ERR_RANGE, "yk_preemption_nodes: NaN node score (zero total on a weighted resource)");
        if (!m) { write_empty(c0, c1); c0 = c1; continue; }
        for (uint32_t r = 0; r < rows; ++r) {
            const uint32_t i = c0 + r;
            const uint32_t* o = e->h_pn_out.p + r * row_words;
            if (k) memcpy(nodes_out + (size_t)i * k, o, 4 * (size_t)k);
            if (k && need_out) memcpy(need_out + (size_t)i * k, o + k, 4 * (size_t)k);
            if (n_fit) n_fit[i] = o[2 * (size_t)k];
            if (best_node) best_node[i] = o[2 * (size_t)k + 1];
            if (best_need) best_need[i] = o[2 * (size_t)k + 2];
        }
        c0 = c1;
    }
    return YK_OK;
}

// Rules 1-2 and 7-8 of the plan run here on the host; rules 3-6 (every bound allocation, every node) on the device.  The host
// repeats rule 5 only on the chosen node's segment and on the headroom step's list, both read back in victim order.
int yk_preemption_plan(yk_engine* e, uint32_t n, const uint32_t* asks, uint32_t* status_out, uint32_t* node_out,
                       uint32_t* victim_off_out, uint32_t* victims_out, uint32_t victims_cap, uint32_t* n_done) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!asks || !status_out || !node_out || !victim_off_out || !n_done))
        return e->fail(YK_ERR_ARG, "yk_preemption_plan: null asks, status_out, node_out, victim_off_out or n_done");
    if (victims_cap && !victims_out) return e->fail(YK_ERR_ARG, "yk_preemption_plan: null victims_out with victims_cap > 0");
    if (!n) { if (n_done) *n_done = 0; if (victim_off_out) victim_off_out[0] = 0; return YK_OK; }
    if (e->pn_seen.size() < e->maxA) { e->pn_seen.assign(e->maxA, 0); e->pn_stamp = 0; }
    if (++e->pn_stamp == 0) { std::fill(e->pn_seen.begin(), e->pn_seen.end(), 0u); e->pn_stamp = 1; }
    for (uint32_t i = 0; i < n; ++i) {
        if (asks[i] >= e->maxA) return e->fail(YK_ERR_ARG, "yk_preemption_plan: ask index beyond max_asks");
        if (e->pn_seen[asks[i]] == e->pn_stamp) return e->fail(YK_ERR_ARG, "yk_preemption_plan: the same ask twice");
        e->pn_seen[asks[i]] = e->pn_stamp;
    }
    int rc = upload_tables(e);
    if (rc) return rc;
    const int D = e->D;
    const uint32_t nlive = e->nlive, nq = e->nq, A = e->a_hi, N = e->maxN;
    cudaStream_t s = e->stream;
    std::vector<uint32_t> order(nlive);
    if (nlive) {   // the cycle's node order, and the NaN check before anything is marked
        CK(grow(e->pn_pos, e->maxN));
        rc = filter_order(e, e->cfg.policy, e->w);
        if (rc) return rc;
        yk_pn_pos_kernel<<<(nlive + 255) / 256, 256, 0, s>>>(e->f_val_out.p, (int)nlive, e->pn_pos.p);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(order.data(), e->f_val_out.p, 4 * (size_t)nlive, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        e->st.other_launches += 1;
        e->st.d2h_bytes += 4 * (size_t)nlive;
        if (e->h_f_flag[0]) return e->fail(YK_ERR_RANGE, "yk_preemption_plan: NaN node score (zero total on a weighted resource)");
    }
    // a plan whose preemptor a cycle has since allocated is spent
    for (uint32_t a = 0; a < A; ++a) if (e->pp_plan[a] != YK_NONE && e->a_state[a] == yk::ST_ALLOCATED) e->pp_plan[a] = YK_NONE;
    const std::vector<uint8_t> mark0 = e->pp_mark;
    const std::vector<uint32_t> plan0 = e->pp_plan;
    auto bail = [&](int code) { e->pp_mark = mark0; e->pp_plan = plan0; return code; };
#define PK(call)                                                                   \
    do {                                                                           \
        cudaError_t _e = (call);                                                   \
        if (_e != cudaSuccess) return bail(e->cuda_fail(_e, #call));               \
    } while (0)

    // ---- queue tables: depth, preorder interval, prefix offsets, guarantee flag, usage for plan calls ----
    const uint32_t* par = e->q_parent.data();
    std::vector<uint32_t> q32(4 * (size_t)nq);   // parent, depth, tin, tout
    uint32_t* depth = q32.data() + nq; uint32_t* tin = depth + nq; uint32_t* tout = tin + nq;
    std::vector<int64_t> q64((size_t)nq * (1 + 2 * D), 0);   // poff, guar, use
    int64_t* poff = q64.data(); int64_t* guar = poff + nq; int64_t* use = guar + (size_t)D * nq;
    std::vector<uint8_t> hasg(nq, 0);
    {
        std::vector<std::vector<uint32_t>> kids(nq);
        for (uint32_t q = 1; q < nq; ++q) kids[par[q]].push_back(q);
        std::vector<std::pair<uint32_t, size_t>> st{{0u, 0}};
        uint32_t clock = 0;
        tin[0] = clock++;
        while (!st.empty()) {   // preorder: q is an ancestor-or-self of x iff tin[q] <= tin[x] < tout[q]
            auto& [q, c] = st.back();
            if (c < kids[q].size()) { const uint32_t ch = kids[q][c++]; tin[ch] = clock++; st.push_back({ch, 0}); }
            else { tout[q] = clock; st.pop_back(); }
        }
    }
    for (uint32_t q = 0; q < nq; ++q) {
        q32[q] = par[q];
        depth[q] = q ? depth[par[q]] + 1 : 0;
        poff[q] = (q ? poff[par[q]] : 0) + e->q_prio_offset[q];
        for (int k = 0; k < D; ++k) {
            guar[(size_t)k * nq + q] = e->q_guar[(size_t)k * nq + q];
            use[(size_t)k * nq + q] = e->q_alloc[(size_t)k * nq + q];
            if (guar[(size_t)k * nq + q] >= 0) hasg[q] = 1;
        }
    }
    auto leaf_of = [&](uint32_t a) { return e->p_queue[e->a_app[a]]; };
    auto req = [&](uint32_t a, int k) { return e->a_req[(size_t)k * e->maxA + a]; };
    auto chain_add = [&](uint32_t a, int sign) {
        for (uint32_t q = leaf_of(a); q != YK_NONE; q = par[q])
            for (int k = 0; k < D; ++k) use[(size_t)k * nq + q] += sign * req(a, k);
    };
    // room for plan calls, and the bound allocations (slots) in ask-index order
    std::vector<int64_t> room((size_t)D * N, 0);
    for (uint32_t x = 0; x < e->n_hi; ++x)
        if (e->n_present[x]) for (int k = 0; k < D; ++k) room[(size_t)k * N + x] = e->n_avail[(size_t)k * N + x];
    std::vector<uint32_t> slot_of(A, YK_NONE), v32, vask, vleaf, vflag, vnode; std::vector<int32_t> vprio; std::vector<uint64_t> ckey;
    for (uint32_t a = 0; a < A; ++a) {
        if (e->pp_mark[a] && e->a_state[a] == yk::ST_ALLOCATED) {
            chain_add(a, -1);
            const uint32_t x = e->a_bound[a];
            if (x < N && e->n_present[x]) for (int k = 0; k < D; ++k) room[(size_t)k * N + x] += req(a, k);
        }
        if (e->pp_plan[a] != YK_NONE && e->a_state[a] != yk::ST_ABSENT) {
            chain_add(a, +1);
            const uint32_t x = e->pp_plan[a];
            if (e->n_present[x]) for (int k = 0; k < D; ++k) room[(size_t)k * N + x] -= req(a, k);
        }
        const uint32_t x = e->a_bound[a];
        if (e->a_state[a] != yk::ST_ALLOCATED || x >= N || !e->n_present[x]) continue;
        slot_of[a] = (uint32_t)vask.size();
        vask.push_back(a); vleaf.push_back(leaf_of(a)); vnode.push_back(x); vprio.push_back(e->a_prio[a]);
        const uint32_t f = e->a_flags[a];
        vflag.push_back(((f & YK_ASK_NO_PREEMPT_SELF) ? YK_PPF_NO_SELF : 0u) | ((f & YK_ASK_ORIGINATOR) ? YK_PPF_ORIGINATOR : 0u) |
                        ((e->a_node[a] != YK_NONE || e->pp_mark[a]) ? YK_PPF_OUT : 0u));
        ckey.push_back(~((uint64_t)e->a_create[a] ^ (1ull << 63)));   // ascending key = create_seq descending
    }
    const uint32_t m = (uint32_t)vask.size();
    if (m >= (1u << 30)) return bail(e->fail(YK_ERR_RANGE, "yk_preemption_plan: 2^30 or more bound allocations"));

    // ---- device tables of the call ----
    const auto bits = [](uint32_t x) { return x ? 32 - __builtin_clz(x) : 0; };
    const int nbits = std::max(1, bits(nlive));   // node keys 0 .. nlive (nlive = not eligible)
    const size_t M = std::max<uint32_t>(m, 1);
    PK(grow(e->pp_q32, q32.size())); PK(grow(e->pp_q64, q64.size())); PK(grow(e->pp_hasg, nq));
    PK(grow(e->pp_v32, 5 * M)); PK(grow(e->pp_vprio, M)); PK(grow(e->pp_taken, M));
    for (int b = 0; b < 2; ++b) { PK(grow(e->pp_key[b], M)); PK(grow(e->pp_tv[b], M)); PK(grow(e->pp_nkey[b], M)); PK(grow(e->pp_nval[b], M)); }
    PK(grow(e->pp_seg, 2 * (size_t)std::max<uint32_t>(nlive, 1))); PK(grow(e->pp_cnt, 1)); PK(grow(e->pp_best, 1));
    PK(grow(e->pp_room, (size_t)D * N)); PK(grow(e->pp_pnode, M + 1)); PK(grow(e->pp_pval, (size_t)D * (M + 1)));
    size_t b1 = 0, b2 = 0;
    PK(cub::DeviceRadixSort::SortPairs(nullptr, b1, e->pp_key[0].p, e->pp_key[1].p, e->pp_tv[0].p, e->pp_tv[1].p, (int)M, 0, 64, s));
    PK(cub::DeviceRadixSort::SortPairs(nullptr, b2, e->pp_nkey[0].p, e->pp_nkey[1].p, e->pp_nval[0].p, e->pp_nval[1].p, (int)M, 0, nbits, s));
    PK(grow(e->pp_cub, std::max(b1, b2)));
    uint32_t* d_ask = e->pp_v32.p; uint32_t* d_leaf = d_ask + M; uint32_t* d_flag = d_leaf + M; uint32_t* d_node = d_flag + M;
    uint32_t* d_perm = d_node + M;
    PK(cudaMemcpyAsync(e->pp_q32.p, q32.data(), 4 * q32.size(), cudaMemcpyHostToDevice, s));
    PK(cudaMemcpyAsync(e->pp_q64.p, q64.data(), 8 * (size_t)nq * (1 + D), cudaMemcpyHostToDevice, s));   // poff, guar
    PK(cudaMemcpyAsync(e->pp_hasg.p, hasg.data(), nq, cudaMemcpyHostToDevice, s));
    PK(cudaMemcpyAsync(e->pp_room.p, room.data(), 8 * room.size(), cudaMemcpyHostToDevice, s));
    e->st.h2d_bytes += 4 * q32.size() + 8 * (size_t)nq * (1 + D) + nq + 8 * room.size();
    std::vector<uint32_t> perm(m);
    if (m) {   // the create-order positions: one stable sort of the slots by create_seq descending (ties: ask index)
        std::vector<uint32_t> iota(m);
        for (uint32_t i = 0; i < m; ++i) iota[i] = i;
        PK(cudaMemcpyAsync(d_ask, vask.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
        PK(cudaMemcpyAsync(d_leaf, vleaf.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
        PK(cudaMemcpyAsync(d_flag, vflag.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
        PK(cudaMemcpyAsync(d_node, vnode.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
        PK(cudaMemcpyAsync(e->pp_vprio.p, vprio.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
        PK(cudaMemcpyAsync(e->pp_key[0].p, ckey.data(), 8 * (size_t)m, cudaMemcpyHostToDevice, s));
        PK(cudaMemcpyAsync(e->pp_tv[0].p, iota.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
        size_t tb = e->pp_cub.n;
        PK(cub::DeviceRadixSort::SortPairs(e->pp_cub.p, tb, e->pp_key[0].p, e->pp_key[1].p, e->pp_tv[0].p, d_perm, (int)m, 0, 64, s));
        PK(cudaMemcpyAsync(perm.data(), d_perm, 4 * (size_t)m, cudaMemcpyDeviceToHost, s));
        PK(cudaStreamSynchronize(s));
        e->st.other_launches += 10;
        e->st.h2d_bytes += 32 * (size_t)m;
        e->st.d2h_bytes += 4 * (size_t)m;
    }
    YkPPArgs pa{};
    pa.D = D;
    pa.q_parent = e->pp_q32.p; pa.q_depth = e->pp_q32.p + nq; pa.q_tin = e->pp_q32.p + 2 * (size_t)nq; pa.q_tout = e->pp_q32.p + 3 * (size_t)nq;
    pa.q_poff = e->pp_q64.p; pa.q_guar = e->pp_q64.p + nq; pa.q_use = e->pp_q64.p + (size_t)nq * (1 + D); pa.q_hasg = e->pp_hasg.p; pa.nq = (int)nq;
    pa.v_ask = d_ask; pa.v_leaf = d_leaf; pa.v_prio = e->pp_vprio.p; pa.v_flag = d_flag; pa.v_node = d_node; pa.perm = d_perm; pa.m = (int)m;
    pa.pos = e->pn_pos.p; pa.sorted = e->f_val_out.p; pa.nlive = (int)nlive; pa.room = e->pp_room.p;
    pa.total = e->d_total.p; pa.ldn = N; pa.taint = e->d_taint.p; pa.label = e->d_label.p; pa.flags = e->d_flags.p;
    pa.a_req = e->d_areq.p; pa.a_tol = e->d_atol.p; pa.a_need = e->d_aneed.p; pa.a_deny = e->d_adeny.p; pa.lda = e->maxA;

    // ---- host side of the rules ----
    std::vector<int64_t> rem((size_t)D * nq, 0);   // what the victims taken for the current preemptor remove, per queue
    std::vector<uint32_t> touched, tstamp(m, 0);
    uint32_t stamp = 0;
    uint32_t L = 0;
    auto rule5 = [&](uint32_t sl) {
        const uint32_t x = vleaf[sl], v = vask[sl], c = yk_pp_lca(par, depth, x, L);
        for (uint32_t q = x; q != c; q = par[q]) {
            if (!hasg[q]) continue;
            for (int k = 0; k < D; ++k) {
                const int64_t gq = guar[(size_t)k * nq + q];
                if (gq >= 0 && use[(size_t)k * nq + q] - rem[(size_t)k * nq + q] - req(v, k) < gq) return false;
            }
        }
        return true;
    };
    auto take = [&](uint32_t sl, std::vector<uint32_t>& out) {
        out.push_back(vask[sl]);
        tstamp[sl] = stamp;
        for (uint32_t q = vleaf[sl]; q != YK_NONE; q = par[q]) {
            touched.push_back(q);
            for (int k = 0; k < D; ++k) rem[(size_t)k * nq + q] += req(vask[sl], k);
        }
    };
    auto user_over = [&](uint32_t a) {
        const uint32_t p = e->a_app[a];
        if (!e->n_ul || e->p_user[p] == YK_NONE) return false;
        for (uint32_t l = 0; l < e->n_ul; ++l) {
            if (e->ul_user[l] != e->p_user[p]) continue;
            bool on_chain = false;
            for (uint32_t q = leaf_of(a); q != YK_NONE && !on_chain; q = par[q]) on_chain = q == e->ul_queue[l];
            if (!on_chain) continue;
            for (int k = 0; k < D; ++k) {
                const int64_t mx = e->ul_max[(size_t)k * e->n_ul + l];
                if (mx >= 0 && e->ul_alloc[(size_t)k * e->n_ul + l] + req(a, k) > mx) return true;
            }
        }
        return false;
    };
    uint32_t voff = 0, done = 0;
    std::vector<uint32_t> pnode; std::vector<int64_t> pval;
    std::vector<uint32_t> seg(2), segv, elig, v6, v7;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t a = asks[i];
        const uint8_t st = e->a_state[a];
        uint32_t status = YK_PP_NO_VICTIMS, node = YK_NONE;
        v6.clear(); v7.clear();
        for (uint32_t q : touched) for (int k = 0; k < D; ++k) rem[(size_t)k * nq + q] = 0;
        touched.clear();
        if (++stamp == 0) { std::fill(tstamp.begin(), tstamp.end(), 0u); stamp = 1; }
        // rule 1: who may preempt
        if (st == yk::ST_ABSENT || (st != yk::ST_NOFIT && st != yk::ST_SKIPPED) || e->pp_plan[a] != YK_NONE) status = YK_PP_NOT_BLOCKED;
        else if (e->a_flags[a] & YK_ASK_NO_PREEMPT_OTHER) status = YK_PP_NOT_ALLOWED;
        else if ((e->a_flags[a] & YK_ASK_SLOWPATH) || e->a_gang[a] != YK_NONE || e->a_node[a] != YK_NONE) status = YK_PP_UNSUPPORTED;
        else if (user_over(a)) status = YK_PP_NOT_ALLOWED;
        else {
            // rule 2: the preemptor's own guarantee
            L = leaf_of(a);
            bool ok = hasg[L] != 0;
            for (uint32_t q = L; q != YK_NONE && ok; q = par[q])
                for (int k = 0; k < D && ok; ++k) {
                    const int64_t gq = guar[(size_t)k * nq + q];
                    if (gq >= 0 && use[(size_t)k * nq + q] + req(a, k) > gq) ok = false;
                }
            if (!ok) status = YK_PP_GUARANTEE;
        }
        if (status == YK_PP_NO_VICTIMS && nlive) {
            // rules 3-6 on the device
            uint32_t fence = 0;
            for (uint32_t q = L; q != YK_NONE; q = par[q]) if (e->q_pp_fence[q]) { fence = q; break; }
            pa.ask = a; pa.leaf = L; pa.fence = fence; pa.prio = e->a_prio[a];
            PK(cudaMemcpyAsync(e->pp_q64.p + (size_t)nq * (1 + D), use, 8 * (size_t)D * nq, cudaMemcpyHostToDevice, s));
            PK(cudaMemsetAsync(e->pp_cnt.p, 0, 4, s));
            PK(cudaMemsetAsync(e->pp_best.p, 0xFF, 8, s));
            e->st.h2d_bytes += 8 * (size_t)D * nq;
            if (m) {
                const unsigned blocks = (m + 255) / 256;
                yk_pp_victim_kernel<<<blocks, 256, 0, s>>>(pa, e->pp_key[0].p, e->pp_tv[0].p, e->pp_cnt.p);
                size_t tb = e->pp_cub.n;
                PK(cub::DeviceRadixSort::SortPairs(e->pp_cub.p, tb, e->pp_key[0].p, e->pp_key[1].p, e->pp_tv[0].p, e->pp_tv[1].p, (int)m, 0, 64, s));
                yk_pp_nodekey_kernel<<<blocks, 256, 0, s>>>(pa, e->pp_key[1].p, e->pp_tv[1].p, e->pp_nkey[0].p, e->pp_nval[0].p);
                tb = e->pp_cub.n;   // stable: a node's entries stay in victim order
                PK(cub::DeviceRadixSort::SortPairs(e->pp_cub.p, tb, e->pp_nkey[0].p, e->pp_nkey[1].p, e->pp_nval[0].p, e->pp_nval[1].p, (int)m, 0, nbits, s));
                e->st.other_launches += 2 + 10 + 2 + (nbits + 7) / 8;
            }
            yk_pp_node_kernel<<<(nlive + 3) / 4, 128, 0, s>>>(pa, e->pp_nkey[1].p, e->pp_nval[1].p, e->pp_taken.p, e->pp_seg.p, e->pp_best.p);
            PK(cudaGetLastError());
            unsigned long long best = 0; uint32_t cnt = 0;
            PK(cudaMemcpyAsync(&best, e->pp_best.p, 8, cudaMemcpyDeviceToHost, s));
            PK(cudaMemcpyAsync(&cnt, e->pp_cnt.p, 4, cudaMemcpyDeviceToHost, s));
            PK(cudaStreamSynchronize(s));
            e->st.other_launches += 1;
            e->st.d2h_bytes += 12;
            if (best != ~0ull) {
                const uint32_t p = (uint32_t)best, need = (uint32_t)(best >> 32);
                node = order[p];
                if (need) {   // the chosen node's victims: its segment again, rule 5 on the host
                    PK(cudaMemcpyAsync(seg.data(), e->pp_seg.p + 2 * (size_t)p, 8, cudaMemcpyDeviceToHost, s));
                    PK(cudaStreamSynchronize(s));
                    segv.resize(seg[1] - seg[0]);
                    PK(cudaMemcpyAsync(segv.data(), e->pp_nval[1].p + seg[0], 4 * segv.size(), cudaMemcpyDeviceToHost, s));
                    PK(cudaStreamSynchronize(s));
                    e->st.d2h_bytes += 8 + 4 * segv.size();
                    int64_t r[8];
                    for (int k = 0; k < D; ++k) r[k] = room[(size_t)k * N + node];
                    for (uint32_t t : segv) {
                        const uint32_t sl = perm[t];
                        if (!rule5(sl)) continue;
                        take(sl, v6);
                        bool fit = true;
                        for (int k = 0; k < D; ++k) { r[k] += req(vask[sl], k); fit = fit && req(a, k) <= std::max<int64_t>(0, r[k]); }
                        if (fit) break;
                    }
                    if (v6.size() != need) return bail(e->fail(YK_ERR_STATE, "yk_preemption_plan: device and host victim walks differ"));
                }
                // rule 7: queues on the path over their max
                auto deficit = [&](uint32_t q) {
                    for (int k = 0; k < D; ++k) {
                        const int64_t mx = e->q_max[(size_t)k * nq + q];
                        if (mx >= 0 && use[(size_t)k * nq + q] - rem[(size_t)k * nq + q] + req(a, k) > mx) return true;
                    }
                    return false;
                };
                std::vector<uint32_t> over;
                for (uint32_t q = L; q != YK_NONE; q = par[q]) if (deficit(q)) over.push_back(q);
                if (!over.empty()) {
                    elig.resize(cnt);
                    if (cnt) PK(cudaMemcpyAsync(elig.data(), e->pp_tv[1].p, 4 * (size_t)cnt, cudaMemcpyDeviceToHost, s));
                    PK(cudaStreamSynchronize(s));
                    e->st.d2h_bytes += 4 * (size_t)cnt;
                    for (uint32_t t : elig) {
                        const uint32_t sl = perm[t];
                        if (tstamp[sl] == stamp) continue;
                        bool under = false;
                        for (uint32_t q : over) under = under || yk_pp_inside(tin, tout, q, vleaf[sl]);
                        if (!under || !rule5(sl)) continue;
                        take(sl, v7);
                        over.erase(std::remove_if(over.begin(), over.end(), [&](uint32_t q) { return !deficit(q); }), over.end());
                        if (over.empty()) break;
                    }
                }
                if (!over.empty()) node = YK_NONE;   // the headroom cannot be freed: no plan
                else status = v6.empty() && v7.empty() ? YK_PP_FITS : YK_PP_PLANNED;
            }
        }
        const uint32_t nv = (uint32_t)(v6.size() + v7.size());
        if (status == YK_PP_PLANNED && (uint64_t)voff + nv > victims_cap) break;   // stops before this ask
        status_out[i] = status;
        node_out[i] = status == YK_PP_PLANNED || status == YK_PP_FITS ? node : YK_NONE;
        victim_off_out[i] = voff;
        if (status == YK_PP_PLANNED) {
            // rule 8: mark, plan, and bring usage, room and the device copies up to date for the next preemptor
            pnode.clear(); pval.clear();
            auto patch = [&](uint32_t x) { pnode.push_back(x); };
            for (const auto* lst : {&v6, &v7})
                for (uint32_t v : *lst) {
                    victims_out[voff++] = v;
                    e->pp_mark[v] = 1;
                    chain_add(v, -1);
                    for (int k = 0; k < D; ++k) room[(size_t)k * N + e->a_bound[v]] += req(v, k);
                    patch(e->a_bound[v]);
                    vflag[slot_of[v]] |= YK_PPF_OUT;
                    PK(cudaMemcpyAsync(d_flag + slot_of[v], &vflag[slot_of[v]], 4, cudaMemcpyHostToDevice, s));
                }
            e->pp_plan[a] = node;
            chain_add(a, +1);
            for (int k = 0; k < D; ++k) room[(size_t)k * N + node] -= req(a, k);
            patch(node);
            std::sort(pnode.begin(), pnode.end());
            pnode.erase(std::unique(pnode.begin(), pnode.end()), pnode.end());
            const size_t np = pnode.size();
            pval.resize((size_t)D * np);
            for (size_t j = 0; j < np; ++j) for (int k = 0; k < D; ++k) pval[(size_t)k * np + j] = room[(size_t)k * N + pnode[j]];
            PK(cudaMemcpyAsync(e->pp_pnode.p, pnode.data(), 4 * np, cudaMemcpyHostToDevice, s));
            PK(cudaMemcpyAsync(e->pp_pval.p, pval.data(), 8 * pval.size(), cudaMemcpyHostToDevice, s));
            yk_apply_avail_kernel<<<(unsigned)((np + 255) / 256), 256, 0, s>>>(D, e->pp_room.p, N, e->pp_pnode.p, e->pp_pval.p, (int)np);
            PK(cudaGetLastError());
            PK(cudaStreamSynchronize(s));   // the staged vectors change with the next preemptor
            e->st.other_launches += 1;
            e->st.h2d_bytes += 4 * (size_t)nv + 4 * np + 8 * pval.size();
        }
        done = i + 1;
    }
#undef PK
    victim_off_out[done] = voff;
    *n_done = done;
    return YK_OK;
}

// The host decides who may preempt (DESIGN.md §2 item 10) and groups the rest by their required node; the device decides every
// group in one pass (csrc/yk_preempt_required.cuh); the host then applies, in the caller's order, the prefix that fits victims_cap.
int yk_preemption_required_node(yk_engine* e, uint32_t n, const uint32_t* asks, uint32_t* status_out, uint32_t* victim_off_out,
                                uint32_t* victims_out, uint32_t victims_cap, uint32_t* n_done) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (n && (!asks || !status_out || !victim_off_out || !n_done))
        return e->fail(YK_ERR_ARG, "yk_preemption_required_node: null asks, status_out, victim_off_out or n_done");
    if (victims_cap && !victims_out) return e->fail(YK_ERR_ARG, "yk_preemption_required_node: null victims_out with victims_cap > 0");
    if (!n) { if (n_done) *n_done = 0; if (victim_off_out) victim_off_out[0] = 0; return YK_OK; }
    if (e->pn_seen.size() < e->maxA) { e->pn_seen.assign(e->maxA, 0); e->pn_stamp = 0; }
    if (++e->pn_stamp == 0) { std::fill(e->pn_seen.begin(), e->pn_seen.end(), 0u); e->pn_stamp = 1; }
    for (uint32_t i = 0; i < n; ++i) {
        if (asks[i] >= e->maxA) return e->fail(YK_ERR_ARG, "yk_preemption_required_node: ask index beyond max_asks");
        if (e->pn_seen[asks[i]] == e->pn_stamp) return e->fail(YK_ERR_ARG, "yk_preemption_required_node: the same ask twice");
        e->pn_seen[asks[i]] = e->pn_stamp;
    }
    int rc = upload_tables(e);
    if (rc) return rc;
    const int D = e->D;
    const uint32_t nq = e->nq, A = e->a_hi, N = e->maxN;
    cudaStream_t s = e->stream;
    // a plan whose preemptor a cycle has since allocated is spent
    for (uint32_t a = 0; a < A; ++a) if (e->pp_plan[a] != YK_NONE && e->a_state[a] == yk::ST_ALLOCATED) e->pp_plan[a] = YK_NONE;
    auto req = [&](uint32_t a, int k) { return e->a_req[(size_t)k * e->maxA + a]; };
    // over the headroom of a queue max on its path or of a user / group limit that applies to it, from what is allocated
    auto over = [&](uint32_t a) {
        const uint32_t p = e->a_app[a];
        for (uint32_t q = e->p_queue[p]; q != YK_NONE; q = e->q_parent[q])
            for (int k = 0; k < D; ++k) {
                const int64_t mx = e->q_max[(size_t)k * nq + q];
                if (mx >= 0 && e->q_alloc[(size_t)k * nq + q] + req(a, k) > mx) return true;
            }
        if (!e->n_ul || e->p_user[p] == YK_NONE) return false;
        for (uint32_t l = 0; l < e->n_ul; ++l) {
            if (e->ul_user[l] != e->p_user[p]) continue;
            bool on_chain = false;
            for (uint32_t q = e->p_queue[p]; q != YK_NONE && !on_chain; q = e->q_parent[q]) on_chain = q == e->ul_queue[l];
            if (!on_chain) continue;
            for (int k = 0; k < D; ++k) {
                const int64_t mx = e->ul_max[(size_t)k * e->n_ul + l];
                if (mx >= 0 && e->ul_alloc[(size_t)k * e->n_ul + l] + req(a, k) > mx) return true;
            }
        }
        return false;
    };
    // ---- host statuses; the rest grouped by node (groups in order of first appearance, call order inside a group) ----
    std::vector<uint32_t> status(n, YK_PP_NO_VICTIMS), grp(N, YK_NONE), gnode, gcnt, pgrp(n, YK_NONE);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t a = asks[i], x = e->a_node[a];
        const uint8_t st = e->a_state[a];
        if ((st != yk::ST_NOFIT && st != yk::ST_SKIPPED) || e->pp_plan[a] != YK_NONE) status[i] = YK_PP_NOT_BLOCKED;
        else if (x == YK_NONE || (e->a_flags[a] & YK_ASK_SLOWPATH) || e->a_gang[a] != YK_NONE) status[i] = YK_PP_UNSUPPORTED;
        else if (over(a)) status[i] = YK_PP_NOT_ALLOWED;
        else if (x < N && e->n_present[x]) {
            if (grp[x] == YK_NONE) { grp[x] = (uint32_t)gnode.size(); gnode.push_back(x); gcnt.push_back(0); }
            pgrp[i] = grp[x];
            ++gcnt[grp[x]];
        }
    }
    const uint32_t G = (uint32_t)gnode.size();
    std::vector<uint32_t> gpoff(G + 1, 0), pask, ppos(n, YK_NONE);
    std::vector<int32_t> pprio;
    for (uint32_t gi = 0; gi < G; ++gi) gpoff[gi + 1] = gpoff[gi] + gcnt[gi];
    const uint32_t P = gpoff[G];
    pask.resize(P); pprio.resize(P);
    {
        std::vector<uint32_t> fill(gpoff.begin(), gpoff.end() - 1);
        for (uint32_t i = 0; i < n; ++i)
            if (pgrp[i] != YK_NONE) { const uint32_t at = fill[pgrp[i]]++; ppos[i] = at; pask[at] = asks[i]; pprio[at] = e->a_prio[asks[i]]; }
    }
    // room(node) for plan calls, and the slots: allocations on a group's node that may ever be victims, in ask-index order
    std::vector<int64_t> room((size_t)D * G);
    for (uint32_t gi = 0; gi < G; ++gi) for (int k = 0; k < D; ++k) room[(size_t)k * G + gi] = e->n_avail[(size_t)k * N + gnode[gi]];
    std::vector<uint32_t> sask, stg, gseg(G + 1, 0);
    std::vector<int32_t> sprio;
    std::vector<uint64_t> ckey;
    for (uint32_t a = 0; a < A; ++a) {
        if (e->pp_plan[a] != YK_NONE && e->a_state[a] != yk::ST_ABSENT && grp[e->pp_plan[a]] != YK_NONE)
            for (int k = 0; k < D; ++k) room[(size_t)k * G + grp[e->pp_plan[a]]] -= req(a, k);
        const uint32_t x = e->a_bound[a];
        if (e->a_state[a] != yk::ST_ALLOCATED || x >= N || grp[x] == YK_NONE) continue;
        if (e->pp_mark[a]) { for (int k = 0; k < D; ++k) room[(size_t)k * G + grp[x]] += req(a, k); continue; }
        if (e->a_node[a] != YK_NONE) continue;
        const uint32_t f = e->a_flags[a];
        const uint32_t type = (f & YK_ASK_ORIGINATOR) ? YK_PRN_TYPE_ORIGINATOR : (f & YK_ASK_NO_PREEMPT_SELF) ? YK_PRN_TYPE_NO_SELF
                                                                                                               : YK_PRN_TYPE_REGULAR;
        sask.push_back(a); sprio.push_back(e->a_prio[a]); stg.push_back(type << 30 | grp[x]);
        ckey.push_back(~((uint64_t)e->a_create[a] ^ (1ull << 63)));   // ascending key = create_seq descending
        ++gseg[grp[x] + 1];
    }
    for (uint32_t gi = 0; gi < G; ++gi) gseg[gi + 1] += gseg[gi];
    const uint32_t m = (uint32_t)sask.size();
    if (m >= (1u << 30) || G >= (1u << 30)) return e->fail(YK_ERR_RANGE, "yk_preemption_required_node: 2^30 or more allocations or nodes");

    // ---- one pass on the device for every group ----
    std::vector<uint32_t> dst(3 * (size_t)P), vout(m);   // status, count, victim offset per preemptor; the victims
    if (G) {
        const size_t M = std::max<uint32_t>(m, 1);
        CK(grow(e->prn_u32, 2 * M + 3 * (size_t)G + 2 + P)); CK(grow(e->prn_i32, M + P)); CK(grow(e->prn_room, (size_t)D * G));
        for (int b = 0; b < 2; ++b) { CK(grow(e->prn_key[b], M)); CK(grow(e->prn_val[b], M)); }
        CK(grow(e->prn_out, 3 * (size_t)P + M)); CK(grow(e->prn_taken, M));
        size_t tb = 0;
        CK(cub::DeviceRadixSort::SortPairs(nullptr, tb, e->prn_key[0].p, e->prn_key[1].p, e->prn_val[0].p, e->prn_val[1].p, (int)M, 0, 64, s));
        CK(grow(e->prn_cub, tb));
        uint32_t* d_sask = e->prn_u32.p; uint32_t* d_stg = d_sask + M; uint32_t* d_gnode = d_stg + M; uint32_t* d_gseg = d_gnode + G;
        uint32_t* d_gpoff = d_gseg + G + 1; uint32_t* d_pask = d_gpoff + G + 1;
        int32_t* d_sprio = e->prn_i32.p; int32_t* d_pprio = d_sprio + M;
        uint32_t* d_st = e->prn_out.p; uint32_t* d_vout = d_st + 3 * (size_t)P;
        CK(cudaMemcpyAsync(d_gnode, gnode.data(), 4 * (size_t)G, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_gseg, gseg.data(), 4 * (size_t)(G + 1), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_gpoff, gpoff.data(), 4 * (size_t)(G + 1), cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_pask, pask.data(), 4 * (size_t)P, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(d_pprio, pprio.data(), 4 * (size_t)P, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(e->prn_room.p, room.data(), 8 * room.size(), cudaMemcpyHostToDevice, s));
        e->st.h2d_bytes += 4 * (3 * (size_t)G + 2 + 2 * (size_t)P) + 8 * room.size();
        YkPRNArgs ra{};
        ra.D = D;
        ra.s_ask = d_sask; ra.s_prio = d_sprio; ra.s_tg = d_stg; ra.m = (int)m;
        ra.g_node = d_gnode; ra.g_seg = d_gseg; ra.g_poff = d_gpoff; ra.g_room = e->prn_room.p; ra.G = (int)G;
        ra.p_ask = d_pask; ra.p_prio = d_pprio;
        ra.total = e->d_total.p; ra.ldn = N; ra.taint = e->d_taint.p; ra.label = e->d_label.p; ra.flags = e->d_flags.p;
        ra.a_req = e->d_areq.p; ra.a_tol = e->d_atol.p; ra.a_need = e->d_aneed.p; ra.a_deny = e->d_adeny.p; ra.lda = e->maxA;
        if (m) {   // the create order, then the victim order inside each group's segment
            std::vector<uint32_t> iota(m);
            for (uint32_t i = 0; i < m; ++i) iota[i] = i;
            CK(cudaMemcpyAsync(d_sask, sask.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(d_stg, stg.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(d_sprio, sprio.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(e->prn_key[0].p, ckey.data(), 8 * (size_t)m, cudaMemcpyHostToDevice, s));
            CK(cudaMemcpyAsync(e->prn_val[0].p, iota.data(), 4 * (size_t)m, cudaMemcpyHostToDevice, s));
            e->st.h2d_bytes += 24 * (size_t)m;
            size_t t1 = e->prn_cub.n;
            CK(cub::DeviceRadixSort::SortPairs(e->prn_cub.p, t1, e->prn_key[0].p, e->prn_key[1].p, e->prn_val[0].p, e->prn_val[1].p, (int)m, 0, 64, s));
            yk_prn_key_kernel<<<(m + 255) / 256, 256, 0, s>>>(ra, e->prn_val[1].p, e->prn_key[0].p, e->prn_val[0].p);
            CK(cudaGetLastError());
            t1 = e->prn_cub.n;
            CK(cub::DeviceRadixSort::SortPairs(e->prn_cub.p, t1, e->prn_key[0].p, e->prn_key[1].p, e->prn_val[0].p, e->prn_val[1].p, (int)m, 0, 64, s));
            e->st.other_launches += 10 + 1 + 10;   // two cub radix sorts of 64-bit keys and the key kernel
        }
        yk_prn_node_kernel<<<(G + 3) / 4, 128, 0, s>>>(ra, e->prn_val[1].p, e->prn_taken.p, d_st, d_st + P, d_st + 2 * (size_t)P, d_vout);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(dst.data(), d_st, 4 * dst.size(), cudaMemcpyDeviceToHost, s));
        if (m) CK(cudaMemcpyAsync(vout.data(), d_vout, 4 * (size_t)m, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        e->st.other_launches += 1;
        e->st.d2h_bytes += 4 * (dst.size() + (size_t)m);
    }

    // ---- the caller-order prefix that fits victims_cap: mark and plan ----
    uint32_t voff = 0, done = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t at = ppos[i];
        const uint32_t st = at == YK_NONE ? status[i] : dst[at];
        const uint32_t cnt = at == YK_NONE ? 0 : dst[P + at];
        if (st == YK_PP_PLANNED && (uint64_t)voff + cnt > victims_cap) break;   // stops before this ask
        status_out[i] = st;
        victim_off_out[i] = voff;
        if (st == YK_PP_PLANNED) {
            for (uint32_t j = 0; j < cnt; ++j) {
                const uint32_t v = vout[dst[2 * (size_t)P + at] + j];
                victims_out[voff++] = v;
                e->pp_mark[v] = 1;
            }
            e->pp_plan[asks[i]] = e->a_node[asks[i]];
        }
        done = i + 1;
    }
    victim_off_out[done] = voff;
    *n_done = done;
    return YK_OK;
}

int yk_set_exchange(yk_engine* e, yk_allgather_fn fn, void* ctx) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    e->xfn = fn; e->xctx = ctx;
    return YK_OK;
}

int yk_peer_export(yk_engine* e, yk_peer_handles* out) {
    if (!e || !out) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    CK(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)out->blob[0], e->slot[0].d_fit.p));
    CK(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)out->blob[1], e->slot[1].d_fit.p));
    CK(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)out->blob[2], e->d_sync.p));
    return YK_OK;
}

int yk_peer_import(yk_engine* e, uint32_t peer, const yk_peer_handles* in) {
    if (!e || !in) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    if (peer >= 8 || peer >= e->cfg.world || peer == e->cfg.rank) return e->fail(YK_ERR_ARG, "yk_peer_import: bad peer rank");
    if (e->peer_open[peer]) return e->fail(YK_ERR_STATE, "yk_peer_import: peer already imported");
    cudaIpcMemHandle_t h[3];
    memcpy(h, in->blob, sizeof(h));
    void* p0 = nullptr; void* p1 = nullptr; void* p2 = nullptr;
    CK(cudaIpcOpenMemHandle(&p0, h[0], cudaIpcMemLazyEnablePeerAccess));
    CK(cudaIpcOpenMemHandle(&p1, h[1], cudaIpcMemLazyEnablePeerAccess));
    CK(cudaIpcOpenMemHandle(&p2, h[2], cudaIpcMemLazyEnablePeerAccess));
    e->peer_fit[0][peer] = (uint32_t*)p0; e->peer_fit[1][peer] = (uint32_t*)p1; e->peer_sync[peer] = (uint32_t*)p2;
    e->peer_open[peer] = true;
    return YK_OK;
}

int yk_peer_enable(yk_engine* e) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    const uint32_t world = e->cfg.world, rank = e->cfg.rank;
    if (world < 2 || world > 8) return e->fail(YK_ERR_ARG, "yk_peer_enable: world must be 2..8");
    for (uint32_t p = 0; p < world; ++p)
        if (p != rank && !e->peer_open[p]) return e->fail(YK_ERR_STATE, "yk_peer_enable: a peer has not been imported");
    e->peer_fit[0][rank] = e->slot[0].d_fit.p; e->peer_fit[1][rank] = e->slot[1].d_fit.p; e->peer_sync[rank] = e->d_sync.p;
    for (Slot& sl : e->slot) CK(cudaMemset(sl.d_fit.p, 0xFF, sl.d_fit.n * sizeof(uint32_t)));   // slots start wiped
    e->p2p = true;
    return YK_OK;
}

int yk_stats(yk_engine* e, yk_stats_t* out) {
    if (!e || !out) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    *out = e->st;
    return YK_OK;
}

int yk_stats_reset(yk_engine* e) {
    if (!e) return YK_ERR_ARG;
    std::lock_guard<std::mutex> g(e->mu);
    e->st = yk_stats_t{};
    return YK_OK;
}

}  // extern "C"
