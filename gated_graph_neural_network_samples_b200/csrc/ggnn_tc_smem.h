// Shared-memory plan of the tile-local wgmma kernel (ggnn_fwd_tc.cuh): plain host arithmetic, so that it can be checked without a GPU.
//
// Layout (compact tiles): h operand | nstages weight slots | ngather gather tiles | cell biases | per-row constants | CSR slice (csr_cache);
// 128-row tiles: h operand | 2 gather tiles | nstages weight slots | cell biases | CSR slice.  An A operand is DP*kgs/4 bytes (hi + lo), a
// weight slot two 64*DP-byte K-step stages, the per-row constants (kgs/16) * (1 + T with edge bias) floats.
#pragma once
#include <algorithm>
#include <cstddef>

namespace ggnn {

struct TcSmemPlan {
    int ngather = 0;       // gather tiles, >= 2
    int nstages = 0;       // weight ring slots; 0: the tile does not fit
    int csr_cache = 0, csr_cap_msgs = 0;
    size_t smem = 0;       // dynamic shared memory of a launch, bytes
};

// avail: the opt-in shared memory per block less the kernel's static part.  max_tile_msgs / max_tile_types: the batch's largest message
// count and largest number of edge types present in one tile.  ngather_request > 0 replaces max_tile_types (GGNN_TC_GATHER_TILES).
//   1. Compact tile-local launches always stage the per-row constants.  The CSR slice (tile-local unweighted graphs) is staged when it fits
//      beside three operand tiles and the two ring slots a worker holds at once.
//   2. Compact tile-local launches gather up to min(max_tile_types, what fits while the ring keeps MIN_RING_GATHER slots) edge types in
//      one pass, never fewer than two; the 128-row and GLOBAL launches keep two gather tiles (their operand tiles are twice as large).
//   3. The rest of the budget goes to the ring, up to max_stages slots.
constexpr int MIN_RING_GATHER = 4;

inline TcSmemPlan tc_smem_plan(int DP, int kgs, int T, bool local, bool unweighted, bool use_bias, int max_tile_msgs, int max_tile_types,
                               size_t avail, int max_stages, int ngather_request) {
    TcSmemPlan r;
    const size_t opb = (size_t)DP * (size_t)kgs / 4, stage = (size_t)DP * 128;
    const size_t ops2 = 3 * opb;                               // h and two gather tiles
    const size_t bias_b = (size_t)3 * DP * sizeof(float) + 64;
    const bool compact = local && kgs == 1024;
    const size_t row_b = compact ? (size_t)(kgs / 16) * (1 + (use_bias ? T : 0)) * sizeof(float) : 0;
    size_t csr_b = 0;
    if (local && unweighted && T <= 16 && max_tile_msgs <= 4096) {
        const int cap = (max_tile_msgs + 15) / 16 * 16;
        const size_t b = (size_t)((128 * T + 1 + 7) & ~7) * 2 + (size_t)cap;
        if (avail >= ops2 + bias_b + row_b + b + 2 * stage) {
            r.csr_cache = 1;
            r.csr_cap_msgs = cap;
            csr_b = b;
        }
    }
    const size_t fixed = bias_b + csr_b + row_b;
    if (avail < ops2 + fixed + 2 * stage) return r;
    r.ngather = 2;
    if (compact) {
        const size_t room = avail >= fixed + MIN_RING_GATHER * stage ? (avail - fixed - MIN_RING_GATHER * stage) / opb : 0;
        const int cap = (int)std::min<size_t>(room > 2 ? room - 1 : 2, 32);   // room counts the h operand too
        const int want = ngather_request > 0 ? ngather_request : max_tile_types;
        r.ngather = std::max(2, std::min(want, cap));
    }
    const size_t ops = (size_t)(1 + r.ngather) * opb;
    r.nstages = (int)std::min<size_t>((size_t)max_stages, (avail - ops - fixed) / stage);
    r.smem = ops + fixed + (size_t)r.nstages * stage;
    return r;
}

}  // namespace ggnn
