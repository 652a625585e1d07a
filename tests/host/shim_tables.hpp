// Test wiring shared by the CPU shims (tests/host/engine_shim.cpp, tests/host/device_shim.cpp): the queue-priority and
// user-limit tables of the next run, and the ordering engine's view of a run's arguments.  Test infrastructure.
#pragma once
#include "../../yunikorn_k8shim_b200/csrc/yk_orderer.hpp"

#include <cstdint>
#include <vector>

// queue priority properties for the next run (priority.offset / priority.policy = fence); NULL = defaults.  Test
// harness convenience: keeps the long argument lists of the run functions unchanged.
static const int32_t* g_q_prio_offset = nullptr;
static const uint8_t* g_q_prio_fence = nullptr;
extern "C" void host_set_queue_priority(const int32_t* offset, const uint8_t* fence) { g_q_prio_offset = offset; g_q_prio_fence = fence; }
// user / group limits for the next run (same convenience): application users, then the entries [D][n] column-major
static const uint32_t* g_p_user = nullptr; static uint32_t g_n_ul = 0;
static const uint32_t* g_ul_queue = nullptr; static const uint32_t* g_ul_user = nullptr;
static const int64_t* g_ul_max = nullptr; static int64_t* g_ul_alloc = nullptr;
extern "C" void host_set_user_limits(const uint32_t* p_user, uint32_t n, const uint32_t* queue, const uint32_t* user, const int64_t* max, int64_t* alloc) {
    g_p_user = p_user; g_n_ul = n; g_ul_queue = queue; g_ul_user = user; g_ul_max = max; g_ul_alloc = alloc;
}
// what each application holds at the start of the next run (same convenience), [D][nP] column-major; NULL = nothing
static const int64_t* g_p_alloc = nullptr;
extern "C" void host_set_app_alloc(const int64_t* p_alloc) { g_p_alloc = p_alloc; }

// What the engine keeps per ask and application besides the run's arguments: every ask pending, every application present
// and holding what host_set_app_alloc gave (nothing by default), and the per-ask cause table (yk::Tables::a_cause) filled
// by yk::ask_cause, as yk_asks_upsert does.
struct ShimTables {
    std::vector<uint8_t> state, present, cause;
    std::vector<int64_t> p_alloc;
};

inline void wire_orderer(yk::Tables& t, ShimTables& s, int D, uint32_t nA, uint32_t nP, uint32_t nQ, const int64_t* a_req,
                         const int32_t* a_prio, const int64_t* a_create, const uint32_t* a_app, const uint32_t* a_flags,
                         const uint32_t* a_gang, const uint32_t* p_queue, const int64_t* p_submit, const uint32_t* q_parent,
                         const int64_t* q_guar, const int64_t* q_max, int64_t* q_alloc, const uint8_t* q_sort) {
    s.state.assign(nA, yk::ST_PENDING); s.present.assign(nP, 1); s.cause.resize(nA);
    if (g_p_alloc) s.p_alloc.assign(g_p_alloc, g_p_alloc + (size_t)D * nP); else s.p_alloc.assign((size_t)D * nP, 0);
    for (uint32_t a = 0; a < nA; ++a) s.cause[a] = yk::ask_cause(D, a_req, nA, a_flags, a);
    t.D = D; t.maxA = nA; t.maxP = nP; t.nq = nQ;
    t.a_req = a_req; t.a_prio = a_prio; t.a_create = a_create; t.a_app = a_app; t.a_flags = a_flags; t.a_gang = a_gang;
    t.a_cause = s.cause.data();
    t.a_state = s.state.data(); t.p_queue = p_queue; t.p_submit = p_submit; t.p_present = s.present.data();
    t.q_parent = q_parent; t.q_guar = q_guar; t.q_max = q_max; t.q_alloc = q_alloc; t.p_alloc = s.p_alloc.data(); t.q_sort = q_sort;
    t.q_prio_offset = g_q_prio_offset; t.q_prio_fence = g_q_prio_fence;
    t.p_user = g_p_user; t.n_ul = g_n_ul; t.ul_queue = g_ul_queue; t.ul_user = g_ul_user; t.ul_max = g_ul_max; t.ul_alloc = g_ul_alloc;
}
