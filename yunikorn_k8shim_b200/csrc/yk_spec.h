// yk_spec.h -- the rules of the speculative round-commit launch, shared by the device (yk_spec.cuh) and the CPU test
// harness (tests/host/spec_shim.cpp).
//
// In a placement-insensitive cycle (one fifo leaf, no max on its chain, no user limit, one priority) the orderer's whole
// pass order is static (yk::Orderer::extend_static): applications by (submit time, application index), each application's
// asks by (create time, ask index), and only the asks that are pending and carry no cause.  The device builds that order
// from its own copies of the ask and application tables while the host is still setting the cycle up, screens it, and
// starts yk_rounds_kernel on it at once when the screen says the host will choose the same thing.  The host still decides
// everything itself (yklt::choose_commit) and adopts the launch only when its first batch and plan equal what the device
// ran; otherwise it aborts the launch and reads nothing it wrote (DESIGN.md §6.3).
//
// The order is two stable radix sorts over every ask index: by create_key, then by app_key (the application's position
// among the applications sorted by submit_key, or past the last position for an ask that is not kept).  The kept asks then
// lead, in pass order.
#pragma once
#include <stdint.h>
#include "yk_score.h"

namespace ykspec {

constexpr uint8_t ST_ALLOCATED = 1, ST_ABSENT = 255;   // yk::ST_* (yk_orderer.hpp)
constexpr uint32_t NONE = 0xFFFFFFFFu;

// device words of one speculation: the round kernel reads [W_STATUS] and [W_COUNT] (ykrd::Args::go)
enum { W_STATUS = 0, W_COUNT, W_KEPT, W_BAD, W_PRIO_MIN, W_PRIO_MAX, W_NOTTOL_LO, W_NOTTOL_HI, W_TAINT_LO, W_TAINT_HI, W_RUN, W_N = 16 };
// W_STATUS: GO, or why the kernel does not start
enum : uint32_t { GO = 0, NO_ROUND = 1, NO_PRIO = 2, NO_RUN = 4, NO_COUNT = 8 };

// ask a enters the cycle's static order: the pending scan keeps it (present, not allocated, its application present) and
// extend_static does not drop it for a cause (slow path, a request that is not strictly positive)
YK_HD bool kept(uint8_t state, uint8_t app_present, uint8_t cause) {
    return state != ST_ABSENT && state != ST_ALLOCATED && app_present != 0 && cause == 0;
}

// yklt::round_eligible for one ask, without the taints: no gang, no required or forbidden labels, no node name.  The taints
// are checked on the union of the kept asks' untolerated bits (W_NOTTOL) against the live nodes' taints (W_TAINT).
YK_HD bool plain(uint32_t gang, uint64_t need, uint64_t deny, uint32_t node) {
    return gang == NONE && need == 0 && deny == 0 && node == NONE;
}

// signed 64-bit time -> unsigned radix key of the same order
YK_HD uint64_t time_key(int64_t v) { return (uint64_t)v ^ 0x8000000000000000ull; }

// int32 priority -> unsigned word of the same order (W_PRIO_MIN / W_PRIO_MAX start at 0xFFFFFFFF / 0)
YK_HD uint32_t prio_word(int32_t p) { return (uint32_t)p ^ 0x80000000u; }

// the second sort's key: the application's position, and maxP (after every position) for an ask that is not kept
YK_HD uint32_t app_key(bool keep, uint32_t pos, uint32_t maxP) { return keep ? pos : maxP; }

// position i > 0 of the order starts a new run of signature ids
YK_HD uint32_t run_break(const uint32_t* order, const uint32_t* sigid, int i) {
    return i > 0 && sigid[order[i]] != sigid[order[i - 1]] ? 1u : 0u;
}

// with brk the inclusive prefix sum of run_break over the order's first n positions: positions [i, i + un_min) hold one
// signature id, so the plan would carry a uniform run (ykun::plan_segments at min_run = un_min)
YK_HD bool long_run_at(const uint32_t* brk, int i, int n, int un_min) {
    return un_min > 0 && i + un_min <= n && brk[i + un_min - 1] == brk[i];
}

// the stretch the kernel takes: the kept asks up to max_bindings
YK_HD uint32_t stretch_len(uint32_t kept_n, uint32_t max_bindings) { return kept_n < max_bindings ? kept_n : max_bindings; }

// The screen, from the reductions in w: W_STATUS and W_COUNT.  GO only when the host's choice can be this launch: every kept
// ask round-eligible, one priority, no uniform run in the stretch, at least rd_min kept asks and a stretch to decide.
YK_HD void decide(uint32_t* w, uint32_t rd_min, uint32_t max_bindings) {
    const uint32_t kn = w[W_KEPT], n = stretch_len(kn, max_bindings);
    const uint64_t nottol = ((uint64_t)w[W_NOTTOL_HI] << 32) | w[W_NOTTOL_LO], taints = ((uint64_t)w[W_TAINT_HI] << 32) | w[W_TAINT_LO];
    uint32_t s = GO;
    if (w[W_BAD] || (nottol & taints)) s |= NO_ROUND;
    if (kn > 0 && w[W_PRIO_MIN] != w[W_PRIO_MAX]) s |= NO_PRIO;
    if (w[W_RUN]) s |= NO_RUN;
    if (kn < rd_min || n == 0) s |= NO_COUNT;
    w[W_STATUS] = s;
    w[W_COUNT] = n;
}

}  // namespace ykspec
