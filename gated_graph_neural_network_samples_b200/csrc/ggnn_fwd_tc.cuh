// Fused GGNN propagation on Hopper tensor cores (wgmma), sm_90a.
//
// One CTA owns a tile of up to 128 node rows.  hidden_size D is padded to DP = roundup(D, 16) <= 128 inside the kernel only.
// Per timestep (sparse:153-216):
//   G1  agg   [128 x DP ]  = sum_t A_t[128 x DP] . W_t          (A_t = per-type sum of gathered source states)
//   G2  gates [128 x 2DP]  = [agg | h] . K_g                     (+ residual pre-product, + b_g, sigmoid)
//   G3  cand  [128 x DP ]  = [agg | r*h] . K_c                   (+ residual pre-product, + b_c, act)
//   h' = u*h + (1-u)*cand
// fp32 accuracy on bf16 tensor cores: every operand is split x = hi + lo (two bf16, 16 mantissa bits) and each
// product is issued as 3 MMAs  Ah.Bh + Ah.Bl + Al.Bh  (the dropped Al.Bl term is 2^-16 relative); "fast" mode
// issues Ah.Bh only.
//
// Warp roles: warps 0-15 = four worker warpgroups, warp 16 = weight producer (on compact tiles warps 16-19, a warpgroup whose registers
// go to the workers: NTHREADS).  Worker warpgroup w owns rows 64*(w%2) .. +64 and
// columns NH*(w/2) .. +NH (NH = DP/2) of every GEMM output -- for the gate GEMM those columns of r AND of u -- so that the node state,
// the gates, the candidate and their epilogues line up element for element in each thread's wgmma accumulator fragment, and the fp32
// master copy of the node states stays in registers for the whole launch (LOCAL mode: the recurrence never leaves the SM).  On compact
// tiles (<= 64 rows) all four warpgroups work on rows 0..63 and split the columns four ways instead (COMPACT_WIDTH), so none of them
// idles on rows that do not exist.  The gathers are row-per-thread over all 16 worker warps (compact tiles with the CSR slice in shared
// memory: one task per real row and 8-column chunk).
//
// Shared memory (ggnn_tc_smem.h): A-operand tiles, each hi+lo in the canonical K-major no-swizzle layout
//   byte(row, k) = part*PART_B + (k/8)*KGS + row*16 + (k%8)*2     (KGS = 16 * allocated rows: 2048, or 1024 for compact <= 64-row tiles)
// -- h, and p.ngather >= 2 gather tiles (A_t of up to ngather edge types at once; tiles 0 and 1 double as the agg and r*h tiles) --, a
// ring of weight slots that the producer thread fills with cp.async.bulk (1-D TMA) from a pre-split, pre-tiled bf16 copy of the weights
// (every worker warp releases every slot), the biases, the tile's per-row constants (compact tiles) and the tile's CSR slice.
// Every mbarrier wait is bounded; on timeout an error code is written and all roles drain.
#pragma once
#include <cuda_bf16.h>

#include "ggnn_common.cuh"
#include "ggnn_wgmma.cuh"

namespace ggnn {
namespace tc {

constexpr int TILE_M = 128;
constexpr int NUM_WORKERS = 512;          // 16 worker warps = 4 warpgroups
constexpr int WARP_PROD = NUM_WORKERS / 32;
// Threads of ggnn_fwd_tc_kernel.  128-row tiles: the workers + one producer warp (17 warps, 96 registers per thread: 5 warps on one SM
// sub-partition).  Compact tiles: the workers + a producer warpgroup (20 warps, also 96 at launch) that hands all but PRODUCER_REGS of
// its registers to the workers (setmaxnreg): 512 * 112 + 128 * 32 = 640 * 96.  The 128-row instances, whose accumulator fragments are
// twice as wide, do not keep a wgmma pipeline even at 112 registers; they issue one weight slot at a time (gemm_narrow_serial).
template <bool COMPACT>
constexpr int NTHREADS = NUM_WORKERS + (COMPACT ? 128 : 32);
constexpr int WORKER_REGS = 112;
constexpr int PRODUCER_REGS = 32;
static_assert(NUM_WORKERS * WORKER_REGS + (NTHREADS<true> - NUM_WORKERS) * PRODUCER_REGS <= NTHREADS<true> * 96, "register file");
constexpr int MAX_STAGES = 10;            // ring slots; a slot holds TWO K-step stages (2 x 64*DP bytes, one bulk copy)

struct TcLayer {
    // pre-split (bf16 hi/lo), pre-tiled weights: one 64*DP-byte stage per K-step (16 rows) of a [K x DP] block
    const uint8_t* w_edge;    // [T*DP/16]       W_t, t-major
    const uint8_t* w_gate;    // [(R+2)*DP/16] x 2 slots: K_g as one N = 2*DP operand (cols r | u): hi slot then lo slot per K-step
                              //                 rows: residual segments..., agg, h
    const uint8_t* w_cand;    // [(R+2)*DP/16]   K_c (RNN: the only kernel)
    const float* edge_b;    // fp32 originals (unpadded)
    const float* gate_b;
    const float* cand_b;
    int steps, nres;
    int res[MAX_RES];
};

struct TcParams {
    int V, D, DP, T, L;
    int use_bias, use_avg, cell, act;
    int save;
    int nparts;   // 3: bf16x3 (fp32-accurate), 1: single bf16 MMA
    int nstages;  // weight ring depth
    int ngather;  // gather tiles (>= 2): the A_t of up to ngather edge types are gathered in one pass, then their MMAs run back to back
    int kgs;            // A-operand k-group stride in bytes: 2048 (128-row tiles) or 1024 (compact: every tile has <= 64 rows)
    int csr_cache;      // LOCAL unweighted only: the tile's CSR slice is staged in shared memory (uint16 row offsets, uint8 local sources)
    int csr_cap_msgs;   // capacity of the shared source array
    const int* tile_start;
    const unsigned* tile_mask;
    const int* row_ptr;
    const int* csr_src;
    const float* slot_w;   // [M] weight of each CSR slot (weighted dense adjacency), or nullptr
    const float* indeg;
    const float* denom;
    const float* state[MAX_LAYERS + 1];
    float* state_w[MAX_LAYERS + 1];
    TcLayer layer[MAX_LAYERS];
    SaveDev save_buf;
    int step_base[MAX_LAYERS];
    float* res_pre;  // [ntiles][128][3*DP] fp32 scratch: residual pre-products of the current layer
    int g_layer, g_step;
    const float* g_in;
    float* g_out;
    float drop_keep;                // state dropout (ggnn_common.cuh dropout_apply); off when >= 1
    unsigned long long drop_seed;
    int* error_flag;
};

// ------------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait (~1 s at 2 GHz).  Returns false on timeout or if another role already aborted.
__device__ __forceinline__ bool mbar_try(uint32_t addr, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                 : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ bool mbar_spin(uint32_t addr, uint32_t parity, volatile int* abort_flag) {
    const long long t0 = clock64();
    for (unsigned it = 1;; ++it) {
        uint32_t ok;
        // the hardware suspends the thread (up to the hint, in ns) instead of spinning; it wakes on barrier events
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                     : "=r"(ok) : "r"(addr), "r"(parity), "r"(20000u) : "memory");
        if (ok) return true;
        if ((it & 63u) == 0u) {   // keep the common iteration tiny
            if (*abort_flag) return false;
            if (clock64() - t0 > 2000000000LL) { *abort_flag = 1; return false; }
        }
    }
}
__device__ __noinline__ bool mbar_wait_slow(uint32_t addr, uint32_t parity, volatile int* abort_flag) { return mbar_spin(addr, parity, abort_flag); }
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, volatile int* abort_flag) {
    const uint32_t addr = smem_u32(bar);
    if (mbar_try(addr, parity)) return true;
    return mbar_wait_slow(addr, parity, abort_flag);
}
// The same wait without a function call, for the weight ring of the tile kernels: a call inside a setmaxnreg region (the compact tile
// kernel's workers) fails register allocation.
__device__ __forceinline__ bool mbar_wait_inline(uint64_t* bar, uint32_t parity, volatile int* abort_flag) {
    const uint32_t addr = smem_u32(bar);
    if (mbar_try(addr, parity)) return true;
    return mbar_spin(addr, parity, abort_flag);
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// generic-proxy shared-memory writes (operand tiles) -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// per-thread register budget of the executing warpgroup from here on (every thread of the warpgroup executes it)
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// x = hi + lo with hi, lo bf16 (round to nearest): 16 mantissa bits kept
__device__ __forceinline__ void split8(const float (&x)[8], uint4& hi, uint4& lo) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const __nv_bfloat162 hp = __floats2bfloat162_rn(x[2 * j], x[2 * j + 1]);   // one packed cvt
        h[j] = *reinterpret_cast<const uint32_t*>(&hp);
        const float r0 = x[2 * j] - __uint_as_float(h[j] << 16);
        const float r1 = x[2 * j + 1] - __uint_as_float(h[j] & 0xFFFF0000u);
        const __nv_bfloat162 lp = __floats2bfloat162_rn(r0, r1);
        l[j] = *reinterpret_cast<const uint32_t*>(&lp);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}
__device__ __forceinline__ void unpack8_add(const uint4& a, float (&acc)[8], float scale) {
    const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        acc[2 * j] = fmaf(scale, __uint_as_float(w[j] << 16), acc[2 * j]);
        acc[2 * j + 1] = fmaf(scale, __uint_as_float(w[j] & 0xFFFF0000u), acc[2 * j + 1]);
    }
}
__device__ __forceinline__ float sigmoid_fast(float v) { return __fdividef(1.0f, 1.0f + __expf(-v)); }
__device__ __forceinline__ float act_fast(float v, int act) {
    return act == ACT_TANH ? (1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * v))) : fmaxf(v, 0.0f);
}

// store one [row, 8-column chunk] of an A operand (both parts)
// (rows at or beyond the allocated row count of a compact tile are not stored: they would alias the next k-group)
__device__ __forceinline__ void store_operand_chunk(uint8_t* op, uint32_t kgs, uint32_t part_b, int kc, int row, const float (&x)[8]) {
    if ((uint32_t)row * 16u >= kgs) return;
    uint4 hi, lo;
    split8(x, hi, lo);
    uint8_t* p = op + (size_t)kc * kgs + (size_t)row * 16;
    *reinterpret_cast<uint4*>(p) = hi;
    *reinterpret_cast<uint4*>(p + part_b) = lo;
}

// ------------------------------------------------------------------------------------------------ the kernel
// 8-wide helpers on [row, 8-column chunk] tiles (the row-per-thread gathers).  D % 4 == 0, so every float4 of a chunk is entirely
// inside or entirely outside the D real columns, and every column pair of an accumulator fragment is.
__device__ __forceinline__ void load8_guarded(const float* base, int col0, int D, float (&v)[8]) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (col0 + 4 <= D) a = *reinterpret_cast<const float4*>(base + col0);
    if (col0 + 8 <= D) b = *reinterpret_cast<const float4*>(base + col0 + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void load8_guarded_cg(const float* base, int col0, int D, float (&v)[8]) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (col0 + 4 <= D) a = __ldcg(reinterpret_cast<const float4*>(base + col0));
    if (col0 + 8 <= D) b = __ldcg(reinterpret_cast<const float4*>(base + col0 + 4));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void store8_guarded(float* base, int col0, int D, const float (&v)[8]) {
    if (col0 + 4 <= D) *reinterpret_cast<float4*>(base + col0) = make_float4(v[0], v[1], v[2], v[3]);
    if (col0 + 8 <= D) *reinterpret_cast<float4*>(base + col0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// one (row, column pair) of an A operand, both parts (split as split8 does); rows at or beyond the allocated row count of a compact tile
// are not stored: they would alias the next k-group
__device__ __forceinline__ void store_operand_pair(uint8_t* op, uint32_t kgs, uint32_t part_b, int row, int col, float x0, float x1) {
    if ((uint32_t)row * 16u >= kgs) return;
    const __nv_bfloat162 hp = __floats2bfloat162_rn(x0, x1);
    const uint32_t h = *reinterpret_cast<const uint32_t*>(&hp);
    const __nv_bfloat162 lp = __floats2bfloat162_rn(x0 - __uint_as_float(h << 16), x1 - __uint_as_float(h & 0xFFFF0000u));
    uint8_t* q = op + (size_t)(col >> 3) * kgs + (size_t)row * 16 + (size_t)(col & 7) * 2;
    *reinterpret_cast<uint32_t*>(q) = h;
    *reinterpret_cast<uint32_t*>(q + part_b) = *reinterpret_cast<const uint32_t*>(&lp);
}
__device__ __forceinline__ void lds8(const float* s, float (&v)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(s), b = *reinterpret_cast<const float4*>(s + 4);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ float2 ld2_cg(const float* p) { return __ldcg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ void st2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }

// ------------------------------------------------------------------------------------------------ the weight ring of the tile kernels
// (this file's kernel and gcn::gcn_wgmma_kernel).  One producer thread streams pre-tiled weights into `nslots` slots of two K-step stages
// (2 x stage_b bytes, one bulk copy); every worker warp takes every slot in push order and releases it once its MMAs are complete.

// tid 0, before the CTA's first __syncthreads: the barriers of all `nslots` slots the kernel declares
__device__ __forceinline__ void ring_init(uint64_t* full, uint64_t* empty, int nslots) {
    for (int i = 0; i < nslots; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], NUM_WORKERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// All-worker rendezvous on hardware named barrier 1; the abort flag is OR-reduced over the barrier so that every worker sees the same
// verdict (ok = false) and all leave together.
__device__ __forceinline__ void workers_sync(volatile int* abortp, bool& ok) {
    uint32_t any;
    asm volatile("{\n\t.reg .pred pa, pb;\n\tsetp.ne.u32 pa, %1, 0;\n\tbar.red.or.pred pb, 1, %2, pa;\n\tselp.u32 %0, 1, 0, pb;\n\t}\n"
                 : "=r"(any) : "r"((uint32_t)(*abortp != 0)), "n"(NUM_WORKERS) : "memory");
    if (any) ok = false;
}

// The consumer side, one per worker thread.
struct RingReader {
    uint64_t* full;           // [nslots] the slot's bytes have landed
    uint64_t* empty;          // [nslots] every worker warp is done with the slot
    volatile int* abortp;
    uint32_t base;            // shared address of slot 0
    uint32_t nslots;
    uint32_t slot = 0, fpar = 0;   // the next slot / bit s: the parity to wait for on full[s]
    // the next slot, its bytes landed (a timeout raises the abort flag and returns the slot anyway: the caller still releases it)
    __device__ __forceinline__ uint32_t take() {
        const uint32_t sl = slot;
        slot = (slot + 1 == nslots) ? 0u : slot + 1;
        if (!*abortp && !mbar_wait_inline(&full[sl], (fpar >> sl) & 1u, abortp)) *abortp = 1;
        fpar ^= 1u << sl;
        return sl;
    }
    __device__ __forceinline__ void release(uint32_t sl, int lane) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[sl]); }
};

// The producer side, one thread, strictly in the order the workers consume.  A slot is refilled once every worker warp has released it,
// so no waiter can be two phases behind a barrier.
struct RingWriter {
    uint64_t* full;
    uint64_t* empty;
    volatile int* abortp;
    uint8_t* base;            // slot 0
    uint32_t nslots, stage_b;
    uint32_t cur = 0, used = 0, epar = 0;   // the next slot / bit s: slot s has been filled before / parity to wait for on empty[s]
    bool ok = true;                         // false after a timeout: nothing more is pushed
    // stream `n` consecutive stage_b-byte stages of a pre-tiled matrix, two per slot
    __device__ __forceinline__ void push(const uint8_t* src, int n) {
        for (int i = 0; i < n && ok; i += 2) {
            const uint32_t bytes = (i + 1 < n) ? 2u * stage_b : stage_b;
            const uint32_t sl = cur;
            cur = (cur + 1 == nslots) ? 0u : cur + 1;
            if ((used >> sl) & 1u) {
                if (!mbar_wait_inline(&empty[sl], (epar >> sl) & 1u, abortp)) { ok = false; break; }
                epar ^= 1u << sl;
            }
            used |= 1u << sl;
            mbar_arrive_expect_tx(&full[sl], bytes);
            bulk_copy_g2s(base + sl * 2u * stage_b, src + (size_t)i * stage_b, bytes, &full[sl]);
        }
    }
};

// After the MMAs of slot i are committed: keep them in flight and release slot i-1 (`prev`) once wgmma.wait_group 1 says its group has
// retired.  A worker warp holds two slots at a time, so the ring has at least two (forward_tc).  `first` is a constant after unrolling:
// a wait_group on a path ptxas cannot resolve makes it serialise every MMA.
__device__ __forceinline__ void retire_slot(RingReader& ring, uint32_t sl, uint32_t& prev, bool first, int lane) {
    if (!first) {
        wg::wait<1>();
        ring.release(prev, lane);
    }
    prev = sl;
}
// the end of a GEMM: every MMA complete (the caller reads the accumulators next, or rewrites an operand tile), the last slot released
__device__ __forceinline__ void retire_last(RingReader& ring, uint32_t prev, int lane) {
    wg::wait_all();
    ring.release(prev, lane);
}

// acc += A(op) . B(one DP x DP weight block: ceil(NKS/2) slots of two K-steps, each stage = [hi | lo]) for one worker warpgroup: A rows from
// byte a_row on (k-group stride KGS, lo part DP*KGS/8 after hi), B columns col0 .. +WN.  X3: three MMAs per product.  Every trip count is a
// template constant (an odd NKS ends in a slot of one K-step), so the MMAs of a slot are straight-line code that ptxas does not serialise.
// Every warpgroup issues its MMAs, also on operand rows that the tile does not have: the operand tiles hold zeros there and the epilogues
// never store those rows.
template <int WN, int DP, bool X3, uint32_t KGS>
__device__ __forceinline__ void gemm_narrow(RingReader& ring, float (&acc)[WN / 2], uint32_t op, uint32_t a_row, int col0, int lane) {
    constexpr int NKS = DP / 16, NSLOTS = (NKS + 1) / 2;
    constexpr uint32_t STAGE_B = DP * 64u, PART_B = DP * KGS / 8u;
    uint32_t prev = 0;
#pragma unroll
    for (int i = 0; i < NSLOTS; ++i) {
        const uint32_t sl = ring.take();
        const uint32_t b0 = ring.base + sl * 2u * STAGE_B + (uint32_t)col0 * 16u;
        wg::fence();
#pragma unroll
        for (int h = 0; h < ((2 * i + 1 < NKS) ? 2 : 1); ++h) {
            const uint32_t a = op + (uint32_t)(2 * i + h) * 2u * KGS + a_row;
            const uint32_t b = b0 + (uint32_t)h * STAGE_B;
            const uint64_t ad = wg::make_desc(a, KGS, 128), bd = wg::make_desc(b, 16u * DP, 128);
            wg::Mma<WN>::run(acc, ad, bd);
            if (X3) {
                wg::Mma<WN>::run(acc, ad, wg::make_desc(b + 32u * DP, 16u * DP, 128));
                wg::Mma<WN>::run(acc, wg::make_desc(a + PART_B, KGS, 128), bd);
            }
        }
        wg::commit();
        retire_slot(ring, sl, prev, i == 0, lane);
    }
    retire_last(ring, prev, lane);
}

// gemm_narrow with A from registers (wgmma RS), for the compact bf16x3 instances: per K-step each warp loads its A_hi and A_lo fragments
// once (ldmatrix) and the three MMAs take A from there, instead of each MMA reading A from shared memory again.  The same MMAs in the same
// order as gemm_narrow, so the sums are bit-identical.  Every K-step is its own wgmma group: wait_group 1 after K-step k retires k-1,
// whose A registers K-step k+1 reuses; slot i is released once its last K-step has retired.  `a_frag` = op + a_row + 16 * 16 * (warp
// in warpgroup) + wg::lds_a_offset(lane, KGS).
template <int WN, int DP, bool X3, uint32_t KGS>
__device__ __forceinline__ void gemm_narrow_rs(RingReader& ring, float (&acc)[WN / 2], uint32_t a_frag, int col0, int lane) {
    constexpr int NKS = DP / 16;
    constexpr uint32_t STAGE_B = DP * 64u, PART_B = DP * KGS / 8u;
    uint32_t sl = 0, prev = 0;
#pragma unroll
    for (int k = 0; k < NKS; ++k) {
        if (k % 2 == 0) sl = ring.take();
        const uint32_t b = ring.base + sl * 2u * STAGE_B + (uint32_t)(k % 2) * STAGE_B + (uint32_t)col0 * 16u;
        const uint32_t a = a_frag + (uint32_t)k * 2u * KGS;
        uint32_t ah[4], al[4];
        wg::ldsm_a(ah, a);
        if (X3) wg::ldsm_a(al, a + PART_B);
        const uint64_t bd = wg::make_desc(b, 16u * DP, 128);
        wg::fence();
        wg::Mma<WN>::run(acc, ah, bd);
        if (X3) {
            wg::Mma<WN>::run(acc, ah, wg::make_desc(b + 32u * DP, 16u * DP, 128));
            wg::Mma<WN>::run(acc, al, bd);
        }
        wg::commit();
        if (k > 0) wg::wait<1>();
        if (k % 2 == 0) {
            if (k > 0) ring.release(prev, lane);   // K-step k-1, the previous slot's last, has retired
            prev = sl;
        }
    }
    retire_last(ring, prev, lane);
}

// The same product one slot at a time (commit, wait for every group, release), for the 128-row layout of ggnn_fwd_tc_kernel: its
// accumulator fragments are twice as wide as the compact ones, ptxas cannot keep a wgmma pipeline under the 96-register cap of 17 warps,
// and an unrolled pipelined body only lengthens live ranges and spills.  A warpgroup without rows (mma_rows false) skips the MMAs but
// still takes and releases every slot.
template <int WN, int DP, bool X3, uint32_t KGS>
__device__ __forceinline__ void gemm_narrow_serial(RingReader& ring, float (&acc)[WN / 2], uint32_t op, uint32_t a_row, int col0, bool mma_rows,
                                                   int lane) {
    constexpr int NKS = DP / 16, NSLOTS = (NKS + 1) / 2;
    constexpr uint32_t STAGE_B = DP * 64u, PART_B = DP * KGS / 8u;
#pragma unroll 1
    for (int i = 0; i < NSLOTS; ++i) {
        const uint32_t sl = ring.take();
        if (mma_rows) {
            const uint32_t b0 = ring.base + sl * 2u * STAGE_B + (uint32_t)col0 * 16u;
            const int nk = (2 * i + 1 < NKS) ? 2 : 1;
            wg::fence();
            for (int h = 0; h < nk; ++h) {
                const uint32_t a = op + (uint32_t)(2 * i + h) * 2u * KGS + a_row;
                const uint32_t b = b0 + (uint32_t)h * STAGE_B;
                const uint64_t ad = wg::make_desc(a, KGS, 128), bd = wg::make_desc(b, 16u * DP, 128);
                wg::Mma<WN>::run(acc, ad, bd);
                if (X3) {
                    wg::Mma<WN>::run(acc, ad, wg::make_desc(b + 32u * DP, 16u * DP, 128));
                    wg::Mma<WN>::run(acc, wg::make_desc(a + PART_B, KGS, 128), bd);
                }
            }
            wg::commit();
            wg::wait_all();
        }
        ring.release(sl, lane);
    }
}

// Column split of the compact layout (tiles of <= 64 rows): all four worker warpgroups on MMA rows 0..63, each with about a quarter of the
// DP = 2*NH output columns.  Every warpgroup computes the same width WC, DP/4 rounded up to a multiple of 8 (the wgmma N), so one body
// serves them all: warpgroup w computes columns min(w*WC, DP-WC) .. +WC and owns -- stores -- those from w*WC on.  DP = 16k, k odd: 4k+4
// columns, the last warpgroup recomputing 8 of its neighbour's (DP = 112: owned 32/32/32/16); at DP = 16 and 48 the last warpgroup owns
// no columns.  The slowest warpgroup's MMA chain is as long as with unequal widths (4k+4, 4k+4, 4k-4, 4k-4).
template <int NH>
constexpr int COMPACT_WIDTH = (NH / 2) % 8 == 0 ? NH / 2 : NH / 2 + 4;

// COMPACT: every tile has <= 64 rows (k-group stride 1024) and the four warpgroups split the columns (COMPACT_WIDTH); otherwise
// warpgroup w owns MMA rows 64*(w%2) .. +64 and columns NH*(w/2) .. +NH.  X3: bf16x3 (p.nparts == 3), else one bf16 MMA per product.
// DP = 2*NH and the k-group stride are template constants too, so that every MMA path is straight-line code.
template <bool LOCAL, int NH, bool COMPACT, bool X3>
__global__ void __launch_bounds__(NTHREADS<COMPACT>, 1) ggnn_fwd_tc_kernel(const __grid_constant__ TcParams p) {
    constexpr int WN = COMPACT ? COMPACT_WIDTH<NH> : NH;   // the columns of one warpgroup (wgmma N, an instruction immediate)
    constexpr int NF = WN / 2;   // accumulator floats per thread and quantity (m64 x WN fragment)
    constexpr int NJ = WN / 8;   // 8-column blocks of a fragment
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ __align__(8) uint64_t bar_full[MAX_STAGES];    // weight slot landed
    __shared__ __align__(8) uint64_t bar_empty[MAX_STAGES];   // every worker warp is done with the slot
    __shared__ int s_abort;

    constexpr int DP = 2 * NH;
    constexpr int NKC = DP >> 3;   // 8-column chunks per DP
    constexpr int NKS = DP >> 4;   // K-steps (16) per DP-wide operand
    constexpr uint32_t KGS = COMPACT ? 1024u : 2048u;   // (p.kgs)
    constexpr uint32_t PART_B = (uint32_t)DP * KGS / 8u;   // bytes per part (hi or lo)
    constexpr uint32_t OPB = 2u * PART_B;                  // bytes per A operand (hi + lo)
    constexpr uint32_t STAGE_B = (uint32_t)DP * 64u;       // bytes per weight stage (K = 16 x N = DP, hi + lo)
    const int D = p.D, T = p.T;
    constexpr int RA = (int)(KGS / 16u);                   // allocated rows of an A operand
    uint8_t* opH = smem;
    // compact: h | ring | ngather gather tiles (the producer's ring at a fixed offset); 128-row: h | 2 gather tiles | ring
    const int ngather = COMPACT ? p.ngather : 2;
    const size_t ring_b = (size_t)p.nstages * 2 * STAGE_B;
    uint8_t* ring = opH + (COMPACT ? 1 : 3) * OPB;                               // nstages slots of 2*STAGE_B, 1024-byte aligned
    uint8_t* opX = COMPACT ? ring + ring_b : opH + OPB;                          // gather tile 0
    uint8_t* opA = opX + OPB;                                                    // gather tile 1
    constexpr bool row_cache = COMPACT;                                          // the per-row constants are staged (compact tiles)
    float* sBias = reinterpret_cast<float*>(COMPACT ? opX + (size_t)ngather * OPB : ring + ring_b);   // [3*DP]: gate r | gate u | cand
    float* sInvDen = sBias + 3 * DP;                                             // [RA] (row_cache): 1/denominator, 1 without averaging
    float* sIndeg = sInvDen + RA;                                                // [RA*T] (row_cache, use_bias): in-degree per type
    uint16_t* sRowPtr = reinterpret_cast<uint16_t*>(sInvDen + (row_cache ? RA * (1 + (p.use_bias ? T : 0)) : 0));   // [128*T + 1] (csr_cache)
    uint8_t* sSrc = reinterpret_cast<uint8_t*>(sRowPtr + ((TILE_M * T + 1 + 7) & ~7)); // [csr_cap_msgs]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.x;
    const int row0 = p.tile_start[tile];
    const int rows = p.tile_start[tile + 1] - row0;
    const unsigned tmask = p.tile_mask[tile];
    const size_t VD = (size_t)p.V * D;
    const int nst = p.nstages;

    if (tid == 0) {
        s_abort = 0;
        ring_init(bar_full, bar_empty, MAX_STAGES);
    }
    __syncthreads();
    volatile int* abortp = &s_abort;

    const int l_begin = LOCAL ? 0 : p.g_layer;
    const int l_end = LOCAL ? p.L : p.g_layer + 1;

    if (warp < WARP_PROD) {
        // =============================================================================== WORKERS
        if (COMPACT) setmaxnreg_inc<WORKER_REGS>();
        // ---- row-per-thread view (gathers): row q*32 + lane, column-chunk group cg
        const int q = warp & 3, cg = warp >> 2;
        const int nkc_tile = NKC;
        constexpr int NCG = NUM_WORKERS / 128;
        const int row = q * 32 + lane;
        // ---- fragment view (GEMMs and epilogues): warpgroup wgi computes rows m0 .. +64, columns col0 .. +WN, and owns those from own0 on
        const int wgi = warp >> 2;
        const int m0 = COMPACT ? 0 : 64 * (wgi & 1);
        const int own0 = COMPACT ? WN * wgi : NH * (wgi >> 1);
        const int col0 = COMPACT ? min(own0, DP - WN) : own0;
        const int fr0 = m0 + (warp & 3) * 16 + (lane >> 2);         // fragment rows fr0, fr0 + 8
        const int fc0 = col0 + (lane & 3) * 2;                      // fragment columns fc0 + 8j, fc0 + 8j + 1
        bool ok = true;
        auto workers_sync = [&]() { tc::workers_sync(abortp, ok); };
        auto publish_sync = [&]() { fence_async_smem(); workers_sync(); };   // operand tiles written -> visible to wgmma
        RingReader rd{bar_full, bar_empty, abortp, smem_u32(ring), (uint32_t)nst};
        const uint32_t a_row = (uint32_t)m0 * 16u;   // this warpgroup's first row inside an A operand
        const bool mma_rows = m0 < rows;             // warpgroup-uniform: the warpgroup has rows at all (always, on compact tiles)
        // Compact tiles pipeline the MMAs (gemm_narrow); 128-row tiles issue one slot at a time (gemm_narrow_serial).  `rs` (a constant
        // at every call): on compact tiles, A from registers -- gemm_narrow_rs at bf16x3 (A_hi feeds two MMAs); a bf16 K-step has one MMA
        // per A, so it stays in shared memory.  The residual pre-products keep A in shared memory: with their three accumulators and the
        // state live, register A makes ptxas serialise every MMA of the NH 56 and 64 instances.
        const uint32_t a_frag = a_row + (uint32_t)(warp & 3) * 256u + wg::lds_a_offset(lane, KGS);   // this warp's ldsm_a offset
        auto gemm_narrow = [&](float (&acc)[NF], const uint8_t* op, bool rs) {
            if constexpr (COMPACT) {
                if (X3 && rs) tc::gemm_narrow_rs<WN, DP, X3, KGS>(rd, acc, smem_u32(op) + a_frag, col0, lane);
                else tc::gemm_narrow<WN, DP, X3, KGS>(rd, acc, smem_u32(op), a_row, col0, lane);
            } else {
                tc::gemm_narrow_serial<WN, DP, X3, KGS>(rd, acc, smem_u32(op), a_row, col0, mma_rows, lane);
            }
        };
        // [r | u] += A(op) . B(one segment of the N = 2*DP gate block: NKS slots, stage 0 = hi, stage 1 = lo); columns of r and of u.
        // One K-step per slot; slot i's MMAs stay in flight while slot i+1's are issued (compact), or one slot at a time (128-row).
        // `rs`, compact tiles: A from registers, at both precisions (every A part feeds the MMAs of r and of u), loaded once per K-step;
        // the same MMAs in the same order.  The group of slot i-1 has retired before slot i+1 reloads the registers (retire_slot's
        // wait_group 1).
        auto wide_mmas = [&](float (&ar)[NF], float (&au)[NF], uint32_t sl, uint32_t a, bool rs) {
            const uint32_t bh = rd.base + sl * 2u * STAGE_B, bl = bh + STAGE_B;
            const uint32_t cr = (uint32_t)col0 * 16u, cu = (uint32_t)(DP + col0) * 16u, lbo = 32u * DP;
            if constexpr (COMPACT) {
                if (rs) {
                    uint32_t ah[4], al[4];
                    wg::ldsm_a(ah, a - a_row + a_frag);
                    if (X3) wg::ldsm_a(al, a - a_row + a_frag + PART_B);
                    wg::fence();
                    wg::Mma<WN>::run(ar, ah, wg::make_desc(bh + cr, lbo, 128));
                    wg::Mma<WN>::run(au, ah, wg::make_desc(bh + cu, lbo, 128));
                    if (X3) {
                        wg::Mma<WN>::run(ar, ah, wg::make_desc(bl + cr, lbo, 128));
                        wg::Mma<WN>::run(au, ah, wg::make_desc(bl + cu, lbo, 128));
                        wg::Mma<WN>::run(ar, al, wg::make_desc(bh + cr, lbo, 128));
                        wg::Mma<WN>::run(au, al, wg::make_desc(bh + cu, lbo, 128));
                    }
                    wg::commit();
                    return;
                }
            }
            const uint64_t ad = wg::make_desc(a, KGS, 128);
            wg::fence();
            wg::Mma<WN>::run(ar, ad, wg::make_desc(bh + cr, lbo, 128));
            wg::Mma<WN>::run(au, ad, wg::make_desc(bh + cu, lbo, 128));
            if (X3) {
                const uint64_t al = wg::make_desc(a + PART_B, KGS, 128);
                wg::Mma<WN>::run(ar, ad, wg::make_desc(bl + cr, lbo, 128));
                wg::Mma<WN>::run(au, ad, wg::make_desc(bl + cu, lbo, 128));
                wg::Mma<WN>::run(ar, al, wg::make_desc(bh + cr, lbo, 128));
                wg::Mma<WN>::run(au, al, wg::make_desc(bh + cu, lbo, 128));
            }
            wg::commit();
        };
        auto gemm_wide = [&](float (&ar)[NF], float (&au)[NF], const uint8_t* op, bool rs) {
            if constexpr (COMPACT) {
                uint32_t prev = 0;
#pragma unroll
                for (int i = 0; i < NKS; ++i) {
                    const uint32_t sl = rd.take();
                    wide_mmas(ar, au, sl, smem_u32(op) + (uint32_t)i * 2u * KGS + a_row, rs);
                    retire_slot(rd, sl, prev, i == 0, lane);
                }
                retire_last(rd, prev, lane);
            } else {
#pragma unroll 1
                for (int i = 0; i < NKS; ++i) {
                    const uint32_t sl = rd.take();
                    if (mma_rows) {
                        wide_mmas(ar, au, sl, smem_u32(op) + (uint32_t)i * 2u * KGS + a_row, rs);
                        wg::wait_all();
                    }
                    rd.release(sl, lane);
                }
            }
        };
        auto zero = [](float (&a)[NF]) {
#pragma unroll
            for (int i = 0; i < NF; ++i) a[i] = 0.0f;
        };
        // fragment element (j, half, e) = acc[4j + 2*half + e]: row fr0 + 8*half, column fc0 + 8j + e.  The epilogues visit the elements
        // of the columns the warpgroup owns only (the others are stored by their owner and never read back by this warpgroup).
#define GGNN_FRAG_PAIRS(...)                                                    \
    _Pragma("unroll") for (int j = 0; j < NJ; ++j)                              \
    _Pragma("unroll") for (int hf = 0; hf < 2; ++hf) {                          \
        const int fi = 4 * j + 2 * hf;                                          \
        const int fr = fr0 + 8 * hf, fc = fc0 + 8 * j;                          \
        const bool fok = fr < rows && fc < D;                                   \
        const int fg = row0 + (fr < rows ? fr : 0);                             \
        (void)fi; (void)fok; (void)fg;                                          \
        if (!COMPACT || fc >= own0) { __VA_ARGS__ }                             \
    }

        // ---- initial state: global fp32 -> registers (fp32 master) + opH (bf16 hi/lo)
        float hs[NF];
        if (COMPACT) zero(hs);   // (the elements of columns the warpgroup does not own are never loaded)
        {
            const float* hin = LOCAL ? p.state[0] : p.g_in;
            GGNN_FRAG_PAIRS({
                float2 v = make_float2(0.f, 0.f);
                if (fok) v = ld2_cg(hin + (size_t)fg * D + fc);
                hs[fi] = v.x; hs[fi + 1] = v.y;
                store_operand_pair(opH, KGS, PART_B, fr, fc, v.x, v.y);
            })
        }
        const bool csr_smem = LOCAL && p.csr_cache && !p.slot_w;   // (the staged slice carries no slot weights)
        if (csr_smem) {
            const int base = p.row_ptr[(size_t)row0 * T];
            const int nptr = rows * T + 1;
            for (int i = tid; i < TILE_M * T + 1; i += NUM_WORKERS) sRowPtr[i] = (uint16_t)(p.row_ptr[(size_t)row0 * T + min(i, nptr - 1)] - base);
            const int mt = p.row_ptr[(size_t)(row0 + rows) * T] - base;
            for (int i = tid; i < mt; i += NUM_WORKERS) sSrc[i] = (uint8_t)(p.csr_src[base + i] - row0);
        }
        // the per-row constants of the agg epilogue, read every timestep: staged once (the same expressions as the epilogue's global reads)
        if (row_cache) {
            for (int i = tid; i < RA; i += NUM_WORKERS) sInvDen[i] = (p.use_avg && i < rows) ? __fdividef(1.0f, p.denom[row0 + i]) : 1.0f;
            if (p.use_bias)
                for (int i = tid; i < RA * T; i += NUM_WORKERS) sIndeg[i] = i < rows * T ? p.indeg[(size_t)row0 * T + i] : 0.0f;
        }
        publish_sync();

        for (int l = l_begin; l < l_end && ok; ++l) {
            const TcLayer& ly = p.layer[l];
            const int s_begin = LOCAL ? 0 : p.g_step;
            const int s_end = LOCAL ? ly.steps : p.g_step + 1;
            const bool gru = p.cell == CELL_GRU;
            // ---- this layer's cell biases -> shared (zero padded to DP)
            for (int i = tid; i < 3 * DP; i += NUM_WORKERS) {
                const int blk = i / DP, col = i - blk * DP;
                float b = 0.0f;
                if (col < D) b = (blk < 2) ? (gru ? ly.gate_b[blk * D + col] : 0.0f) : ly.cand_b[col];
                sBias[i] = b;
            }
            workers_sync();
            // ---- residual pre-products (constant over the layer's timesteps): Pg = res . K_g[res rows], Pc = res . K_c[res rows]
            float* res_pre = p.res_pre + (size_t)tile * TILE_M * 3 * DP;
            if (ly.nres > 0 && s_end > s_begin) {
                float pr[NF], pu[NF], pc[NF];
                zero(pr); zero(pu); zero(pc);
                for (int i = 0; i < ly.nres && ok; ++i) {
                    const float* rs = p.state[ly.res[i]];
                    GGNN_FRAG_PAIRS({
                        float2 v = make_float2(0.f, 0.f);
                        if (fok) v = ld2_cg(rs + (size_t)fg * D + fc);
                        store_operand_pair(opA, KGS, PART_B, fr, fc, v.x, v.y);
                    })
                    publish_sync();
                    if (!ok) break;
                    if (gru) gemm_wide(pr, pu, opA, false);
                    gemm_narrow(pc, opA, false);
                    workers_sync();   // opA is rewritten next
                }
                GGNN_FRAG_PAIRS({
                    float* d = res_pre + (size_t)fr * 3 * DP + fc;
                    st2(d, pr[fi], pr[fi + 1]); st2(d + DP, pu[fi], pu[fi + 1]); st2(d + 2 * DP, pc[fi], pc[fi + 1]);
                })
            }
            for (int s = s_begin; s < s_end && ok; ++s) {
                const size_t save_base = (size_t)(p.step_base[l] + s) * VD;
                // ------------------------------------------------------------ gather + G1
                // Compact tiles: the A_t of a group of present types are gathered into consecutive gather tiles (rotating over the ngather
                // tiles), published with one barrier, then the group's MMAs run back to back in type order, so acc sums the same products in
                // the same order as one type at a time.  A tile whose types fit in the gather tiles is one group; otherwise groups of
                // ngather/2 types, so that a group never overwrites the tiles of the group before it, whose MMAs other warpgroups may still
                // be issuing.  128-row tiles: one type at a time, A_t alternating between opA and opX (the gather of type n+1 never
                // overwrites what the MMAs of type n read).
                float acc[NF];
                zero(acc);
                const int gsz = __popc(tmask) <= ngather ? ngather : ngather / 2;   // (compact)
                int nty = 0, n = 0, gt = 0, gt0 = 0;   // types gathered; of them in the open group; the next gather tile; the group's first
                unsigned grp = 0u;   // (compact, CSR slice in shared memory) the open group's types, gathered when it closes
                // The gather touches shared memory only, so with compact tiles -- rows 0..63 only -- all 16 worker warps share it:
                // row group = warp & 1, eight column-chunk groups instead of four.
                const bool gsplit = KGS == 1024u;
                const int g_row = gsplit ? ((warp & 1) * 32 + lane) : row;
                const bool g_row_ok = g_row < rows;
                const int g_grow = g_row_ok ? row0 + g_row : row0;
                const int g_cg = gsplit ? (warp >> 1) : cg, g_ncg = gsplit ? NUM_WORKERS / 64 : NCG;
                const int g_nkc = gsplit ? nkc_tile : (((uint32_t)(q * 32) * 16u < KGS) ? nkc_tile : 0);
                for (int t = 0; t < T && ok; ++t) {
                    if (!((tmask >> t) & 1u)) continue;
                    if (n == 0) gt0 = gt;
                    uint8_t* gdst = COMPACT ? opX + (size_t)gt * OPB : ((nty & 1) ? opX : opA);
                    gt = gt + 1 == ngather ? 0 : gt + 1;
                    ++nty;
                    ++n;
                    if (COMPACT && csr_smem) {
                        grp |= 1u << t;
                    } else {
                        int beg = 0, end = 0;
                        if (g_row_ok) {
                            if (csr_smem) { beg = sRowPtr[g_row * T + t]; end = sRowPtr[g_row * T + t + 1]; }
                            else { beg = p.row_ptr[(size_t)g_grow * T + t]; end = p.row_ptr[(size_t)g_grow * T + t + 1]; }
                        }
                        for (int kc = g_cg; kc < g_nkc; kc += g_ncg) {
                            float a8[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j) a8[j] = 0.0f;
                            if (LOCAL && csr_smem) {
                                // fast path: local source indices from shared memory, two messages in flight
                                const uint8_t* colbase = opH + (size_t)kc * KGS;
                                const uint32_t lo_off = PART_B;
                                int m = beg;
                                if (X3) {
                                    for (; m + 1 < end; m += 2) {
                                        const uint8_t* s0 = colbase + (size_t)sSrc[m] * 16;
                                        const uint8_t* s1 = colbase + (size_t)sSrc[m + 1] * 16;
                                        const uint4 h0 = *reinterpret_cast<const uint4*>(s0), l0 = *reinterpret_cast<const uint4*>(s0 + lo_off);
                                        const uint4 h1 = *reinterpret_cast<const uint4*>(s1), l1 = *reinterpret_cast<const uint4*>(s1 + lo_off);
                                        unpack8_add(h0, a8, 1.0f); unpack8_add(h1, a8, 1.0f);
                                        unpack8_add(l0, a8, 1.0f); unpack8_add(l1, a8, 1.0f);
                                    }
                                    if (m < end) {
                                        const uint8_t* s0 = colbase + (size_t)sSrc[m] * 16;
                                        unpack8_add(*reinterpret_cast<const uint4*>(s0), a8, 1.0f);
                                        unpack8_add(*reinterpret_cast<const uint4*>(s0 + lo_off), a8, 1.0f);
                                    }
                                } else {
                                    for (; m < end; ++m) unpack8_add(*reinterpret_cast<const uint4*>(colbase + (size_t)sSrc[m] * 16), a8, 1.0f);
                                }
                            } else {
                                // each message scaled by its slot weight (a weighted dense adjacency) or by 1: fmaf(1, x, y) rounds as x + y
                                for (int m = beg; m < end; ++m) {
                                    if (LOCAL) {
                                        const float a = p.slot_w ? p.slot_w[m] : 1.0f;
                                        const uint8_t* sp = opH + (size_t)kc * KGS + (size_t)(p.csr_src[m] - row0) * 16;
                                        unpack8_add(*reinterpret_cast<const uint4*>(sp), a8, a);
                                        if (X3) unpack8_add(*reinterpret_cast<const uint4*>(sp + PART_B), a8, a);
                                    } else {
                                        // GLOBAL mode: source rows come from the previous step's fp32 state in L2; keep 4 rows in flight (each
                                        // weight is read at its accumulate step, not beside the row loads)
                                        float hv[4][8];
                                        const int nb = min(4, end - m);
#pragma unroll
                                        for (int qq = 0; qq < 4; ++qq)
                                            if (qq < nb) load8_guarded_cg(p.g_in + (size_t)p.csr_src[m + qq] * D, kc * 8, D, hv[qq]);
#pragma unroll
                                        for (int qq = 0; qq < 4; ++qq)
                                            if (qq < nb) {
                                                const float a = p.slot_w ? p.slot_w[m + qq] : 1.0f;
#pragma unroll
                                                for (int j = 0; j < 8; ++j) a8[j] = fmaf(a, hv[qq][j], a8[j]);
                                            }
                                        m += nb - 1;
                                    }
                                }
                            }
                            store_operand_chunk(gdst, KGS, PART_B, kc, g_row, a8);
                        }
                    }
                    if (COMPACT && n < gsz && ((tmask >> t) >> 1) != 0) continue;   // the group is open and another type follows
                    if (COMPACT && csr_smem) {
                        // One task per (real row, 8-column chunk), spread over all 512 worker threads, rows fastest (a warp's stores
                        // are contiguous); a task sums the messages of each of the group's types in turn into its gather tile, in the
                        // order of the row-per-thread loop (CSR order, a pair added h0, h1, l0, l1, the odd message last).  Pad rows
                        // (>= rows) of the gather tiles are not written and may hold anything, NaN included: wgmma output row i reads
                        // A row i only, so they reach pad rows of acc only, which the agg epilogue replaces by 0 (v0 = fr < rows ? ... :
                        // 0); every operand of the gate and candidate GEMMs (opX, opA, opH) thus has finite pad rows, and so has hs.
                        const int dk = NUM_WORKERS / rows, dr = NUM_WORKERS - dk * rows;   // task += 512 in (chunk, row); rows >= 1
                        for (int kc = tid / rows, trow = tid - kc * rows; kc < NKC;) {
                            const uint16_t* rp = sRowPtr + trow * T;
                            const uint8_t* colbase = opH + (size_t)kc * KGS;
                            int j = gt0;
                            for (unsigned g = grp; g != 0u; g &= g - 1u) {
                                const int tg = __ffs(g) - 1;
                                float a8[8];
#pragma unroll
                                for (int e = 0; e < 8; ++e) a8[e] = 0.0f;
                                int m = rp[tg];
                                const int end = rp[tg + 1];
                                if (X3) {
                                    for (; m + 1 < end; m += 2) {
                                        const uint8_t* s0 = colbase + (size_t)sSrc[m] * 16;
                                        const uint8_t* s1 = colbase + (size_t)sSrc[m + 1] * 16;
                                        const uint4 h0 = *reinterpret_cast<const uint4*>(s0), l0 = *reinterpret_cast<const uint4*>(s0 + PART_B);
                                        const uint4 h1 = *reinterpret_cast<const uint4*>(s1), l1 = *reinterpret_cast<const uint4*>(s1 + PART_B);
                                        unpack8_add(h0, a8, 1.0f); unpack8_add(h1, a8, 1.0f);
                                        unpack8_add(l0, a8, 1.0f); unpack8_add(l1, a8, 1.0f);
                                    }
                                    if (m < end) {
                                        const uint8_t* s0 = colbase + (size_t)sSrc[m] * 16;
                                        unpack8_add(*reinterpret_cast<const uint4*>(s0), a8, 1.0f);
                                        unpack8_add(*reinterpret_cast<const uint4*>(s0 + PART_B), a8, 1.0f);
                                    }
                                } else {
                                    for (; m < end; ++m) unpack8_add(*reinterpret_cast<const uint4*>(colbase + (size_t)sSrc[m] * 16), a8, 1.0f);
                                }
                                store_operand_chunk(opX + (size_t)j * OPB, KGS, PART_B, kc, trow, a8);
                                j = j + 1 == ngather ? 0 : j + 1;
                            }
                            kc += dk;
                            trow += dr;
                            if (trow >= rows) { trow -= rows; ++kc; }
                        }
                        grp = 0u;
                    }
                    publish_sync();
                    if (!ok) break;
                    if constexpr (COMPACT) {
                        for (int k = 0, j = gt0; k < n; ++k, j = (j + 1 == ngather) ? 0 : j + 1) gemm_narrow(acc, opX + (size_t)j * OPB, true);
                    } else {
                        gemm_narrow(acc, gdst, false);
                    }
                    n = 0;
                }
                workers_sync();   // every G1 MMA is complete before the gather tiles (opX / opA) are rewritten
                if (!ok) break;
                // ------------------------------------------------------------ agg epilogue: + indeg.B, / (deg + 1e-7) -> opX
                GGNN_FRAG_PAIRS({
                    float v0 = acc[fi], v1 = acc[fi + 1];
                    if (p.use_bias && fc < D) {
                        for (int t = 0; t < T; ++t) {
                            const float ind = row_cache ? sIndeg[fr * T + t] : p.indeg[(size_t)fg * T + t];
                            const float2 b = *reinterpret_cast<const float2*>(ly.edge_b + (size_t)t * D + fc);
                            v0 = fmaf(ind, b.x, v0); v1 = fmaf(ind, b.y, v1);
                        }
                    }
                    const float inv_den = row_cache ? sInvDen[fr] : (p.use_avg && fr < rows) ? __fdividef(1.0f, p.denom[fg]) : 1.0f;
                    v0 = fr < rows ? v0 * inv_den : 0.0f;
                    v1 = fr < rows ? v1 * inv_den : 0.0f;
                    if (p.save && fok) st2(p.save_buf.agg + save_base + (size_t)fg * D + fc, v0, v1);
                    store_operand_pair(opX, KGS, PART_B, fr, fc, v0, v1);
                })
                publish_sync();
                if (!ok) break;
                float* outp = LOCAL ? ((s == ly.steps - 1) ? p.state_w[l + 1] : nullptr) : p.g_out;
                if constexpr (COMPACT) {
                    // one candidate GEMM for both cells: a second copy under a runtime branch keeps ptxas from pipelining the MMAs
                    float gu[NF];   // GRU: the update gate u
                    if (gru) {
                        // -------------------------------------------------------- gates: r*h -> opA, u stays in registers
                        float gr[NF];
                        zero(gr); zero(gu);
                        gemm_wide(gr, gu, opX, true);
                        gemm_wide(gr, gu, opH, true);
                        GGNN_FRAG_PAIRS({
                            float br0 = sBias[fc], br1 = sBias[fc + 1], bu0 = sBias[DP + fc], bu1 = sBias[DP + fc + 1];
                            if (ly.nres > 0) {
                                const float* rp = res_pre + (size_t)fr * 3 * DP + fc;
                                br0 += rp[0]; br1 += rp[1]; bu0 += rp[DP]; bu1 += rp[DP + 1];
                            }
                            const float r0 = sigmoid_fast(gr[fi] + br0), r1 = sigmoid_fast(gr[fi + 1] + br1);
                            gu[fi] = sigmoid_fast(gu[fi] + bu0); gu[fi + 1] = sigmoid_fast(gu[fi + 1] + bu1);
                            if (p.save && fok) {
                                const size_t o = save_base + (size_t)fg * D + fc;
                                st2(p.save_buf.r + o, r0, r1);
                                st2(p.save_buf.h_in + o, hs[fi], hs[fi + 1]);
                                st2(p.save_buf.u + o, gu[fi], gu[fi + 1]);
                            }
                            store_operand_pair(opA, KGS, PART_B, fr, fc, r0 * hs[fi], r1 * hs[fi + 1]);
                        })
                        publish_sync();
                        if (!ok) break;
                    }
                    // ------------------------------------------------------------ candidate [agg | r*h] . K_c (GRU), [agg | h] . K_c (RNN); new state
                    float gc[NF];
                    zero(gc);
                    gemm_narrow(gc, opX, true);
                    gemm_narrow(gc, gru ? opA : opH, true);
                    GGNN_FRAG_PAIRS({
                        float bc0 = sBias[2 * DP + fc], bc1 = sBias[2 * DP + fc + 1];
                        if (ly.nres > 0) {
                            const float* rp = res_pre + (size_t)fr * 3 * DP + 2 * DP + fc;
                            bc0 += rp[0]; bc1 += rp[1];
                        }
                        if (gru) {
                            const float c0 = act_fast(gc[fi] + bc0, p.act), c1 = act_fast(gc[fi + 1] + bc1, p.act);
                            if (p.save && fok) st2(p.save_buf.c + save_base + (size_t)fg * D + fc, c0, c1);
                            gc[fi] = fmaf(gu[fi], hs[fi] - c0, c0);            // u*h + (1-u)*c
                            gc[fi + 1] = fmaf(gu[fi + 1], hs[fi + 1] - c1, c1);
                        } else {
                            if (p.save && fok) st2(p.save_buf.h_in + save_base + (size_t)fg * D + fc, hs[fi], hs[fi + 1]);
                            gc[fi] = act_fast(gc[fi] + bc0, p.act);
                            gc[fi + 1] = act_fast(gc[fi + 1] + bc1, p.act);
                        }
                    })
#pragma unroll
                    for (int i = 0; i < NF; ++i) hs[i] = gc[i];
                } else {
                    if (gru) {
                        // -------------------------------------------------------- gates: r*h -> opA, u stays in registers
                        float gr[NF], gu[NF];
                        zero(gr); zero(gu);
                        gemm_wide(gr, gu, opX, false);
                        gemm_wide(gr, gu, opH, false);
                        GGNN_FRAG_PAIRS({
                            float br0 = sBias[fc], br1 = sBias[fc + 1], bu0 = sBias[DP + fc], bu1 = sBias[DP + fc + 1];
                            if (ly.nres > 0) {
                                const float* rp = res_pre + (size_t)fr * 3 * DP + fc;
                                br0 += rp[0]; br1 += rp[1]; bu0 += rp[DP]; bu1 += rp[DP + 1];
                            }
                            const float r0 = sigmoid_fast(gr[fi] + br0), r1 = sigmoid_fast(gr[fi + 1] + br1);
                            gu[fi] = sigmoid_fast(gu[fi] + bu0); gu[fi + 1] = sigmoid_fast(gu[fi + 1] + bu1);
                            if (p.save && fok) {
                                const size_t o = save_base + (size_t)fg * D + fc;
                                st2(p.save_buf.r + o, r0, r1);
                                st2(p.save_buf.h_in + o, hs[fi], hs[fi + 1]);
                                st2(p.save_buf.u + o, gu[fi], gu[fi + 1]);
                            }
                            store_operand_pair(opA, KGS, PART_B, fr, fc, r0 * hs[fi], r1 * hs[fi + 1]);
                        })
                        publish_sync();
                        if (!ok) break;
                        // -------------------------------------------------------- candidate, new state
                        float gc[NF];
                        zero(gc);
                        gemm_narrow(gc, opX, false);
                        gemm_narrow(gc, opA, false);
                        GGNN_FRAG_PAIRS({
                            float bc0 = sBias[2 * DP + fc], bc1 = sBias[2 * DP + fc + 1];
                            if (ly.nres > 0) {
                                const float* rp = res_pre + (size_t)fr * 3 * DP + 2 * DP + fc;
                                bc0 += rp[0]; bc1 += rp[1];
                            }
                            const float c0 = act_fast(gc[fi] + bc0, p.act), c1 = act_fast(gc[fi + 1] + bc1, p.act);
                            if (p.save && fok) st2(p.save_buf.c + save_base + (size_t)fg * D + fc, c0, c1);
                            gc[fi] = fmaf(gu[fi], hs[fi] - c0, c0);            // u*h + (1-u)*c
                            gc[fi + 1] = fmaf(gu[fi + 1], hs[fi + 1] - c1, c1);
                        })
#pragma unroll
                        for (int i = 0; i < NF; ++i) hs[i] = gc[i];
                    } else {
                        float gc[NF];
                        zero(gc);
                        gemm_narrow(gc, opX, false);
                        gemm_narrow(gc, opH, false);
                        GGNN_FRAG_PAIRS({
                            float bc0 = sBias[2 * DP + fc], bc1 = sBias[2 * DP + fc + 1];
                            if (ly.nres > 0) {
                                const float* rp = res_pre + (size_t)fr * 3 * DP + 2 * DP + fc;
                                bc0 += rp[0]; bc1 += rp[1];
                            }
                            if (p.save && fok) st2(p.save_buf.h_in + save_base + (size_t)fg * D + fc, hs[fi], hs[fi + 1]);
                            gc[fi] = act_fast(gc[fi] + bc0, p.act);
                            gc[fi + 1] = act_fast(gc[fi + 1] + bc1, p.act);
                        })
#pragma unroll
                        for (int i = 0; i < NF; ++i) hs[i] = gc[i];
                    }
                }
                // Every MMA that reads opH must be complete before the state update rewrites it.  On compact GRU tiles they are already:
                // each warpgroup's gate GEMM, the last reader, drained before the barrier after the gate epilogue, and the candidate reads
                // opX and opA only.  (Writing the state from the candidate epilogue instead keeps more of it live there and spills more.)
                if (!COMPACT || !gru) {
                    workers_sync();
                    if (!ok) break;
                }
                GGNN_FRAG_PAIRS({
                    if (p.drop_keep < 1.0f) {
                        hs[fi] = dropout_apply(hs[fi], p.drop_seed, p.step_base[l] + s, p.V, D, fg, fc, p.drop_keep);
                        hs[fi + 1] = dropout_apply(hs[fi + 1], p.drop_seed, p.step_base[l] + s, p.V, D, fg, fc + 1, p.drop_keep);
                    }
                    store_operand_pair(opH, KGS, PART_B, fr, fc, hs[fi], hs[fi + 1]);
                    if (outp && fok) st2(outp + (size_t)fg * D + fc, hs[fi], hs[fi + 1]);
                })
                publish_sync();   // opH complete before anyone gathers from it
            }  // steps
            if (LOCAL && ok && ly.steps == 0) {   // a layer without timesteps aliases the previous state (sparse:152)
                GGNN_FRAG_PAIRS({
                    if (fok) st2(p.state_w[l + 1] + (size_t)fg * D + fc, hs[fi], hs[fi + 1]);
                })
            }
            if (LOCAL && l + 1 < l_end) { __threadfence(); workers_sync(); }   // layer output visible before it is read as a residual
        }  // layers
#undef GGNN_FRAG_PAIRS
        if (!ok && tid == 0) atomicExch(p.error_flag, 1);
    } else if (COMPACT) {
        setmaxnreg_dec<PRODUCER_REGS>();
    }
    if (warp == WARP_PROD && lane == 0) {
        // =============================================================================== WEIGHT PRODUCER
        // the weights of every layer and step, in the order the workers' GEMMs consume them
        RingWriter wr{bar_full, bar_empty, abortp, ring, (uint32_t)nst, STAGE_B};
        for (int l = l_begin; l < l_end && wr.ok; ++l) {
            const TcLayer& ly = p.layer[l];
            const int s_begin = LOCAL ? 0 : p.g_step;
            const int s_end = LOCAL ? ly.steps : p.g_step + 1;
            const bool gru = p.cell == CELL_GRU;
            const size_t blk = (size_t)NKS * STAGE_B;   // one DP x DP block; a gate block is two of these per K segment
            if (ly.nres > 0 && s_end > s_begin) {
                for (int i = 0; i < ly.nres && wr.ok; ++i) {
                    if (gru) wr.push(ly.w_gate + (size_t)i * 2 * blk, 2 * NKS);
                    wr.push(ly.w_cand + (size_t)i * blk, NKS);
                }
            }
            const size_t kx = (size_t)ly.nres, kh = (size_t)ly.nres + 1;
            for (int s = s_begin; s < s_end && wr.ok; ++s) {
                for (int t = 0; t < T && wr.ok; ++t) {
                    if (!((tmask >> t) & 1u)) continue;
                    wr.push(ly.w_edge + (size_t)t * blk, NKS);
                }
                if (gru) { wr.push(ly.w_gate + kx * 2 * blk, 2 * NKS); wr.push(ly.w_gate + kh * 2 * blk, 2 * NKS); }
                wr.push(ly.w_cand + kx * blk, NKS); wr.push(ly.w_cand + kh * blk, NKS);
            }
        }
        if (!wr.ok) atomicExch(p.error_flag, 3);
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------ weight pre-tiling
// fp32 row-major W[(nseg*D) rows][src_ld cols], columns [src_col0, src_col0 + nblk*D)  ->  per K-step s (16 padded rows) nblk consecutive ring slots of
// 64*DP bytes.  Np = nblk*DP output rows (column block b of the source lands at n = b*DP + col, zero padded):
//   nblk == 1:  slot = [hi part | lo part], part = 2 K-chunks x DP rows x 16 B            (one DP-wide weight block)
//   nblk == 2:  slot 0 = hi part, slot 1 = lo part, part = 2 K-chunks x 2*DP rows x 16 B  (the [r | u] gate block)
// element: byte(s, part, c, n, j) = s*nblk*64*DP + part*(32*Np) + c*(16*Np) + n*16 + j*2 = bf16 part of W[row(s*16+c*8+j)][col(n)]
__global__ void ggnn_tile_weights_kernel(const float* __restrict__ W, uint8_t* __restrict__ out, int D, int DP, int nseg, int nblk,
                                         int src_ld, int src_col0) {
    const int Np = nblk * DP;
    const int ksteps = nseg * DP / 16;
    const long long total = (long long)ksteps * 2 * Np;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(idx % Np);
        const int c = (int)((idx / Np) % 2);
        const int s = (int)(idx / (2 * Np));
        const int blk = n / DP, nn = n - blk * DP;
        float x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int kp = s * 16 + c * 8 + j;
            const int seg = kp / DP, kk = kp - seg * DP;
            x[j] = (kk < D && nn < D) ? W[(size_t)(seg * D + kk) * src_ld + src_col0 + blk * D + nn] : 0.0f;
        }
        uint4 hi, lo;
        split8(x, hi, lo);
        uint8_t* base = out + (size_t)s * nblk * 64 * DP + (size_t)c * 16 * Np + (size_t)n * 16;
        *reinterpret_cast<uint4*>(base) = hi;
        *reinterpret_cast<uint4*>(base + (size_t)32 * Np) = lo;
    }
}

}  // namespace tc
}  // namespace ggnn
