// Streaming GGNN propagation on Hopper tensor cores (wgmma), sm_90a: the path for hidden sizes whose
// per-tile operands do not fit one SM (D > 128, BASELINE config 4) and for batches / graphs too large for the
// tile-local fused kernel (ggnn_fwd_tc.cuh).
//
// One timestep (sparse:153-216) = three launches of ONE kernel template, each a 128-row x NC-column output tile
// per CTA whose K dimension is streamed through a shared-memory ring, KS K-steps (16 columns) per stage:
//   EPI_AGG   agg       = [A_0 | .. | A_{T-1}] . [W_0; ..; W_{T-1}]      A_t[v] = sum of h[src] over the type-t messages into v,
//                         + indeg.B, / (deg + 1e-7)                       gathered by the worker warps straight into the ring (GATHER):
//                         a (target, type) pair with ONE message is a 64-byte asynchronous copy (cp.async, completion on the stage's
//                         mbarrier) of the source row's image chunks, a pair with none is zeros, and the few pairs with several
//                         messages are summed once per launch into "virtual rows" (prologue) and then copied like the others --
//                         no load latency sits between two K-steps of a gather warp.  In a weighted batch every pair whose messages are
//                         not one of weight 1 is a virtual row, summed with its slot weights; with propagation attention every pair
//                         with messages is a virtual row, weighted by the step's probabilities (attention_chunk_kernel, launched first)
//   EPI_GATE  [r | u]   = sigmoid([res.. | agg | h] . K_g + b_g)          writes r*h (operand image) and u
//   EPI_CAND  h'        = u*h + (1-u)*act([res.. | agg | r*h] . K_c + b_c) (RNN: act([res.. | agg | h] . K + b))
// CudnnCompatibleGRUCell (sparse:105-108) applies the reset gate after the recurrent product, so a timestep is four launches:
//   EPI_GATE  as above, but writes r itself (chunk-major fp32) instead of the r*h image
//   EPI_HPROJ q         = h . K_hid + b_hid                                  saves q, overwrites the r chunk with r*q
//   EPI_CAND  h'        = u*h + (1-u)*tanh([res.. | agg] . K_in + b_in + r*q)
// The sparse GCN's streaming plan (ggnn_gcn.cuh, gcn_gather_image_kernel) uses the TMA-fed instance for its layer GEMM:
//   EPI_GCN   H'        = S . W_l + b_l, then relu and state dropout on every layer but the last    S = A . H, gathered into an image
// Node-state operands live in HBM/L2 as bf16 hi/lo "images" in the canonical K-major no-swizzle layout, tile-major:
//   byte(tile, kstep, part, kgroup, row, j) = ((tile*NKS + kstep)*2 + part)*4096 + kgroup*2048 + row*16 + j*2
// so one K-step of a 128-row A operand (hi + lo) is ONE contiguous 8 KB bulk copy (cp.async.bulk, 1-D TMA), and an
// epilogue thread (one row) writes 16-byte chunks that are contiguous across the warp.  Weights are
// pre-split and pre-tiled per (N block, K-step) into contiguous 64*NC-byte stages (ggnn_tile_weights_stream_kernel).
// fp32 accuracy on bf16 tensor cores as in ggnn_fwd_tc.cuh: x = hi + lo, product = Ah.Bh + Ah.Bl + Al.Bh (3 MMAs).
//
// The fp32 master copy of every state (and the update gate u) is kept in a second, chunk-major layout
//   float(tile, chunk = col/8, row, j) = ((tile*NKC + chunk)*128 + row)*8 + j
// so that an epilogue warp (32 rows x 8 columns) reads and writes 1 KB contiguous instead of 32 scattered sectors;
// the user-visible row-major [V, D] arrays are written only for node_states_per_layer entries and for the backward pass.
//
// Roles: warps 0 .. NWORK-1 = workers (gather groups of 4 warps in the edge kernel; epilogue: row = 32*(warp % 4) + lane, column
// group = warp / 4), warps NWORK .. NWORK+7 = two MMA warpgroups (wgmma m64 x MMA_N, one 64-row half of the tile each, accumulators
// in registers; the K-steps per stage and the number of MMAs per product are template parameters, so the wgmma chain of a stage is
// straight-line code and one stage's MMAs stay in flight while the next stage is awaited), warp NWORK+8 = producer (one thread: bulk
// copies).  One thread per MMA warpgroup polls each ring barrier, the rest of the warpgroup waits on a named barrier behind it.  When
// the K loop is done the MMA warpgroups park the accumulator in shared memory over the now idle ring, and the workers' epilogue reads
// it from there.  Every mbarrier wait is bounded; on timeout an error code is written.
#pragma once
#include "ggnn_fwd_tc.cuh"

namespace ggnn {
namespace ts {

using tc::smem_u32;

constexpr int TILE_M = 128;
constexpr int MAX_SEG = MAX_RES + 2;
constexpr int MAX_NS = 8;            // ring stages
constexpr int A_STAGE_B = 8192;      // one K-step of a 128-row A operand: 2 parts x 2 k-groups x 128 rows x 16 B
constexpr int MMA_N = 128;           // output columns per CTA (the wgmma N): 64 fp32 accumulator registers per MMA thread
constexpr int ACC_LD = MMA_N + 4;    // row stride (floats) of the accumulator parked in shared memory: conflict-free float4 rows
constexpr int NWORK = 8;             // worker warps: two gather groups of 128 rows, two epilogue column groups (17 warps in all:
                                     // five per SM sub-partition leave 96 registers per thread)
constexpr int NGATHER = NWORK / 4;   // gather groups (4 warps = 128 rows each)
constexpr int NTHREADS = (NWORK + 9) * 32;
// The shallowest ring the kernel accepts.  The MMA warpgroups keep one stage's MMAs in flight while they await the next, so a ring needs
// two stages.  And a parity wait is only sound if the waiter cannot be two phases ahead of the barrier: a gather group waiting for round r
// of a stage has (through its previous stage, NGATHER stages back) only seen round r-2 complete when the ring has at least as many stages
// as there are gather groups.
constexpr int MIN_NS = 2;
static_assert(NGATHER <= MIN_NS && MIN_NS <= MAX_NS, "every gather group needs a ring stage of its own");
// shared memory of the ring: the stages, and at least the parked accumulator
__host__ __device__ inline size_t ring_bytes(size_t nstages, size_t stage_b) {
    const size_t acc_b = (size_t)TILE_M * ACC_LD * sizeof(float);
    return nstages * stage_b > acc_b ? nstages * stage_b : acc_b;
}
enum { EPI_AGG = 0, EPI_GATE = 1, EPI_CAND = 2, EPI_HPROJ = 3, EPI_GCN = 4 };

struct StreamParams {
    int V, D, DP, T;
    int NC;                // output columns per CTA (== MMA_N); grid.y = number of N blocks
    int nstages;           // ring depth
    int nparts;            // 3: bf16x3, 1: single bf16 MMA
    int epi;               // EPI_*
    int cell, act, use_bias, use_avg;
    // ---- A operand, TMA-fed: nseg K segments, each a DP-wide tile-major image
    int nseg;
    const uint8_t* seg[MAX_SEG];
    // ---- A operand, gathered (EPI_AGG): per present edge type a DP-wide segment of per-type source sums
    const uint8_t* g_img;        // image of the state the messages are gathered from (a row with one type-t message is a 64-byte copy)
    const unsigned* tile_mask;   // [ntiles] bit t: some row of the tile receives a type-t message
    const int* pair_src;         // [ntiles*128*T] per (target, type): -1 no message | source node (exactly one message, of weight 1) | -(2 + vid)
                                 // several, or one of another weight
    const int* vrow_ptr;         // [NV+1] messages of the pairs with several messages (their "virtual rows"), CSR over vid ...
    const int* vsrc;             // ... source nodes in message order
    const int4* vinfo;           // [NV][2]: {count, src0, src1, src2 | src3 .. src6}: the first sources inline, one 32-byte load per virtual row
    const int* tile_vptr;        // [ntiles+1] vid range of each tile
    uint8_t* virt_img;           // image rows of the virtual rows (written in the prologue of every launch, row index = vid)
    const float* slot_w;         // weighted batches: [M] target-CSR slot weights (attention: the step's probabilities), or null (binary:
                                 // every message weighs 1) ...
    const int* vslot;            // ... and [NV] the first slot of every virtual row: message m of virtual row vid weighs slot_w[vslot[vid] + m]
    // ---- B operand
    const uint8_t* w;            // [nblk][kt_all] stages of 64*NC bytes: [hi: 2 k-groups x NC x 16 B | lo: same]
    int kt_all;                  // K-steps per N block in `w`
    // ---- epilogue
    const float* bias;           // AGG: edge_biases [T][D] or null; GATE: gate_bias [2D]; CAND: cand_bias [D]
    const float* indeg;          // [V][T]
    const float* denom;          // [V]
    const float* h_chk;          // fp32 state entering the step, chunk-major   (GATE: r*h, save; CAND: blend)
    float* u_buf;                // update gate, chunk-major: written by GATE, read by CAND
    float* h_chk_out;            // CAND: new state fp32, chunk-major
    float* h_out;                // CAND: new state fp32 row-major [V][D], or null (only node_states_per_layer entries need it)
    float* sv_u;                 // GATE: row-major copy of u for the backward pass, or null
    uint8_t* img_out;            // AGG: agg image; GATE: r*h image; CAND: image of the new state
    float* sv_h; float* sv_agg; float* sv_r; float* sv_c;   // this step's save-for-backward slots or null
    // ---- CudnnCompatibleGRUCell
    const float* b_hid;          // HPROJ: cand_hidden_bias [D]
    float* rq_chk;               // chunk-major fp32: r (written by GATE), r*q (HPROJ), read by CAND
    float* sv_q;                 // HPROJ: row-major save slot of q = h . K_hid + b_hid, or null
    // ---- GCN (EPI_GCN): bias = b_l or null, h_out = H_{l+1} row-major [V][D]
    int relu_dropout;            // relu, then state dropout (every layer but the last)
    float drop_keep; unsigned long long drop_seed; int gstep;
    int* error_flag;
};

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

__device__ __forceinline__ size_t chunk_off(int NKC, int tile, int c, int row) { return (((size_t)tile * NKC + c) * TILE_M + row) * 8; }
__device__ __forceinline__ void chunk_load(const float* base, int NKC, int tile, int c, int row, float (&v)[8]) {
    const float4* q = reinterpret_cast<const float4*>(base + chunk_off(NKC, tile, c, row));
    const float4 a = __ldcg(q), b = __ldcg(q + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void chunk_store(float* base, int NKC, int tile, int c, int row, const float (&v)[8]) {
    float4* q = reinterpret_cast<float4*>(base + chunk_off(NKC, tile, c, row));
    q[0] = make_float4(v[0], v[1], v[2], v[3]);
    q[1] = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void unpack8(const uint4& a, float (&x)[8]) {
    const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { x[2 * j] = __uint_as_float(w[j] << 16); x[2 * j + 1] = __uint_as_float(w[j] & 0xFFFF0000u); }
}

// one [row, 8 columns] chunk of an image (both parts); col0 % 8 == 0
__device__ __forceinline__ void img_store_chunk(uint8_t* img, int NKS, int tile, int row, int col0, const float (&x)[8]) {
    uint4 hi, lo;
    tc::split8(x, hi, lo);
    uint8_t* p = img + ((size_t)tile * NKS + (col0 >> 4)) * A_STAGE_B + (size_t)((col0 >> 3) & 1) * 2048 + (size_t)row * 16;
    *reinterpret_cast<uint4*>(p) = hi;
    *reinterpret_cast<uint4*>(p + 4096) = lo;
}

// Sum of the image rows of one (target, type) pair with several messages, one K-step (16 columns), fp32 in message order, re-split:
// (hi k-group 0, hi k-group 1, lo k-group 0, lo k-group 1).  `info` = vinfo[2*vid..]: {count, src0..src6}; longer lists continue in vsrc.
__device__ __forceinline__ void sum_pair_sources(const uint8_t* __restrict__ g_img, int NKS, int ks, const int4& i0, const int4& i1,
                                                 const int* __restrict__ vsrc_tail, uint4& h0, uint4& h1, uint4& l0, uint4& l1) {
    auto img_row = [&](int src) { return g_img + ((size_t)(src >> 7) * NKS + ks) * A_STAGE_B + (size_t)(src & 127) * 16; };
    float a0[8], a1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { a0[j] = 0.0f; a1[j] = 0.0f; }
    auto add_row = [&](const uint8_t* sp) {
        const uint4 y0 = __ldcg(reinterpret_cast<const uint4*>(sp)), y1 = __ldcg(reinterpret_cast<const uint4*>(sp + 2048));
        const uint4 y2 = __ldcg(reinterpret_cast<const uint4*>(sp + 4096)), y3 = __ldcg(reinterpret_cast<const uint4*>(sp + 6144));
        tc::unpack8_add(y0, a0, 1.0f); tc::unpack8_add(y2, a0, 1.0f);
        tc::unpack8_add(y1, a1, 1.0f); tc::unpack8_add(y3, a1, 1.0f);
    };
    const int cnt = i0.x;
    {   // the first two sources are always there: request both before the first add
        const uint8_t* s0 = img_row(i0.y);
        const uint8_t* s1 = img_row(i0.z);
        const uint4 x0 = __ldcg(reinterpret_cast<const uint4*>(s0)), x1 = __ldcg(reinterpret_cast<const uint4*>(s0 + 2048));
        const uint4 x2 = __ldcg(reinterpret_cast<const uint4*>(s0 + 4096)), x3 = __ldcg(reinterpret_cast<const uint4*>(s0 + 6144));
        const uint4 y0 = __ldcg(reinterpret_cast<const uint4*>(s1)), y1 = __ldcg(reinterpret_cast<const uint4*>(s1 + 2048));
        const uint4 y2 = __ldcg(reinterpret_cast<const uint4*>(s1 + 4096)), y3 = __ldcg(reinterpret_cast<const uint4*>(s1 + 6144));
        tc::unpack8_add(x0, a0, 1.0f); tc::unpack8_add(x2, a0, 1.0f);
        tc::unpack8_add(x1, a1, 1.0f); tc::unpack8_add(x3, a1, 1.0f);
        tc::unpack8_add(y0, a0, 1.0f); tc::unpack8_add(y2, a0, 1.0f);
        tc::unpack8_add(y1, a1, 1.0f); tc::unpack8_add(y3, a1, 1.0f);
    }
    if (cnt > 2) add_row(img_row(i0.w));
    if (cnt > 3) add_row(img_row(i1.x));
    if (cnt > 4) add_row(img_row(i1.y));
    if (cnt > 5) add_row(img_row(i1.z));
    if (cnt > 6) add_row(img_row(i1.w));
    for (int m = 7; m < cnt; ++m) add_row(img_row(vsrc_tail[m]));   // rare tail, in message order
    tc::split8(a0, h0, l0);
    tc::split8(a1, h1, l1);
}

// The same for a weighted batch's virtual row, which may have a single message: sum of w_m * (hi + lo) of its source rows, fp32 fmaf in
// CSR order, hi part then lo part of each row (the accumulation order of the tile kernel's weighted gather).  `w` = its slot weights.
__device__ __forceinline__ void sum_pair_sources_weighted(const uint8_t* __restrict__ g_img, int NKS, int ks, const int4& i0, const int4& i1,
                                                          const int* __restrict__ vsrc_tail, const float* __restrict__ w, uint4& h0, uint4& h1,
                                                          uint4& l0, uint4& l1) {
    float a0[8], a1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { a0[j] = 0.0f; a1[j] = 0.0f; }
    auto add_row = [&](int src, float wm) {
        const uint8_t* sp = g_img + ((size_t)(src >> 7) * NKS + ks) * A_STAGE_B + (size_t)(src & 127) * 16;
        const uint4 y0 = __ldcg(reinterpret_cast<const uint4*>(sp)), y1 = __ldcg(reinterpret_cast<const uint4*>(sp + 2048));
        const uint4 y2 = __ldcg(reinterpret_cast<const uint4*>(sp + 4096)), y3 = __ldcg(reinterpret_cast<const uint4*>(sp + 6144));
        tc::unpack8_add(y0, a0, wm); tc::unpack8_add(y2, a0, wm);
        tc::unpack8_add(y1, a1, wm); tc::unpack8_add(y3, a1, wm);
    };
    const int cnt = i0.x;
    const int inl[7] = {i0.y, i0.z, i0.w, i1.x, i1.y, i1.z, i1.w};
#pragma unroll
    for (int m = 0; m < 7; ++m)
        if (m < cnt) add_row(inl[m], __ldg(w + m));
    for (int m = 7; m < cnt; ++m) add_row(vsrc_tail[m], __ldg(w + m));   // rare tail, in message order
    tc::split8(a0, h0, l0);
    tc::split8(a1, h1, l1);
}

// KS = K-steps (16 columns) per ring stage, a divisor of DP / 16; X3 = three MMAs per product (bf16x3) instead of one
template <bool GATHER, bool X3, int KS>
__global__ void __launch_bounds__(NTHREADS, 1) ggnn_stream_kernel(const __grid_constant__ StreamParams p) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t bar_full[MAX_NS];    // B (and TMA-fed A) bytes landed
    __shared__ __align__(8) uint64_t bar_afull[MAX_NS];   // gathered A written (GATHER)
    __shared__ __align__(8) uint64_t bar_empty[MAX_NS];   // the MMAs that read the stage are complete
    __shared__ __align__(8) uint64_t bar_acc;             // the accumulator is parked in shared memory
    __shared__ int s_abort;
    __shared__ int s_types[32];
    __shared__ int s_ntypes;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.x, nb0 = blockIdx.y;   // the N block of this CTA
    const int D = p.D, DP = p.DP, T = p.T, NC = p.NC, NS = p.nstages;
    const int NKS = DP >> 4;
    const int GPS = NKS / KS;                        // stages ("K groups") per K segment
    const int row0 = tile * TILE_M;
    const int rows = min(TILE_M, p.V - row0);
    const uint32_t B_STEP_B = 64u * (uint32_t)NC;    // one K-step of the B operand: [hi: 2 k-groups x NC x 16 B | lo: same]
    const uint32_t A_REGION_B = (uint32_t)KS * A_STAGE_B;
    const uint32_t STAGE_B = A_REGION_B + (uint32_t)KS * B_STEP_B;   // a stage = KS K-steps of A, then KS K-steps of B
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    int* sPair = reinterpret_cast<int*>(smem + ring_bytes(NS, STAGE_B));   // [128*T] the tile's slice of pair_src (GATHER)
    float* accs = reinterpret_cast<float*>(smem);                         // [128][ACC_LD] parked accumulator (after the K loop)

    if (tid == 0) {
        s_abort = 0;
        for (int i = 0; i < MAX_NS; ++i) { tc::mbar_init(&bar_full[i], 1); tc::mbar_init(&bar_afull[i], TILE_M); tc::mbar_init(&bar_empty[i], 8); }
        tc::mbar_init(&bar_acc, 256);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        int n = 0;
        if (GATHER) {
            const unsigned m = p.tile_mask[tile];
            for (int t = 0; t < T; ++t) if ((m >> t) & 1u) s_types[n++] = t;
        }
        s_ntypes = n;
    }
    __syncthreads();
    volatile int* abortp = &s_abort;
    const int nsegs = GATHER ? s_ntypes : p.nseg;    // K segments of this tile (present edge types / operand images)
    const int ng = nsegs * GPS;                        // stages to stream
    const int nk = nsegs * NKS;                        // K-steps in total

    if (warp == NWORK + 8) {
        // =============================================================================== PRODUCER (one thread)
        // Issuing a bulk copy costs this thread several hundred cycles whatever its size, so a stage carries KS K-steps: the A operand of
        // those K-steps is ONE contiguous piece of the image, their B operand ONE contiguous piece of the pre-tiled weights.
        if (lane == 0) {
            bool ok = true;
            int s = 0, round = 0;
            const uint8_t* wb = p.w + (size_t)nb0 * p.kt_all * B_STEP_B;
            int sg = 0, j = 0;
            for (int g = 0; g < ng && ok; ++g) {
                if (round > 0 && !tc::mbar_wait(&bar_empty[s], (uint32_t)(round - 1) & 1u, abortp)) { ok = false; break; }
                const int ks0 = j * KS, nks = KS;
                uint8_t* st = smem + (size_t)s * STAGE_B;
                const int seg_k0 = (GATHER ? s_types[sg] : sg) * NKS + ks0;   // first K-step of the stage in the weight stream
                if (GATHER) {
                    tc::mbar_arrive_expect_tx(&bar_full[s], (uint32_t)nks * B_STEP_B);
                } else {
                    tc::mbar_arrive_expect_tx(&bar_full[s], (uint32_t)nks * ((uint32_t)A_STAGE_B + B_STEP_B));
                    tc::bulk_copy_g2s(st, p.seg[sg] + ((size_t)tile * NKS + ks0) * A_STAGE_B, (uint32_t)nks * A_STAGE_B, &bar_full[s]);
                }
                tc::bulk_copy_g2s(st + A_REGION_B, wb + (size_t)seg_k0 * B_STEP_B, (uint32_t)nks * B_STEP_B, &bar_full[s]);
                // K order: TMA-fed kernels walk segment by segment; the gather GEMM walks K group by K group over all edge types
                if (GATHER) { if (++sg == nsegs) { sg = 0; ++j; } }
                else if (++j == GPS) { j = 0; ++sg; }
                if (++s == NS) { s = 0; ++round; }
            }
            if (!ok) atomicExch(p.error_flag, 13);
        }
    } else if (warp >= NWORK) {
        // =============================================================================== MMA WARPGROUPS
        // warpgroup m: rows 64*m .. +64 of the tile x MMA_N columns.  Stage g's MMAs are committed as one group; the group of stage g-1 is
        // then awaited (at most one in flight) and stage g-1 released (one arrival per warp).
        constexpr int NF = MMA_N / 2;
        float acc[NF];
#pragma unroll
        for (int i = 0; i < NF; ++i) acc[i] = 0.0f;
        const int m = (warp - NWORK) >> 2;
        const bool poller = ((tid - NWORK * 32) & 127) == 0;
        const uint32_t smem_a = smem_u32(smem) + (uint32_t)m * 1024u;   // this half's first row inside an A stage
        const uint32_t smem_b = smem_u32(smem);
        const uint32_t lbo_b = 16u * (uint32_t)MMA_N;
        int s = 0, prev = -1;
        uint32_t par = 0;
        for (int g = 0; g < ng; ++g) {
            if (poller && !*abortp && !tc::mbar_wait(&bar_full[s], par, abortp)) *abortp = 1;
            if (GATHER && poller && !*abortp && !tc::mbar_wait(&bar_afull[s], par, abortp)) *abortp = 1;
            asm volatile("bar.sync %0, 128;" ::"r"(6 + m) : "memory");
            if (GATHER) tc::fence_async_smem();   // the gathered A stage was written through the generic proxy (cp.async / st.shared)
            const uint32_t a0 = smem_a + (uint32_t)s * STAGE_B, b0 = smem_b + (uint32_t)s * STAGE_B + A_REGION_B;
            wg::fence();
#pragma unroll
            for (int i = 0; i < KS; ++i) {
                const uint32_t a = a0 + (uint32_t)i * A_STAGE_B, b = b0 + (uint32_t)i * B_STEP_B;
                const uint64_t ah = wg::make_desc(a, 2048, 128), bh = wg::make_desc(b, lbo_b, 128);
                wg::Mma<MMA_N>::run(acc, ah, bh);
                if (X3) {
                    wg::Mma<MMA_N>::run(acc, ah, wg::make_desc(b + 32u * MMA_N, lbo_b, 128));
                    wg::Mma<MMA_N>::run(acc, wg::make_desc(a + 4096u, 2048, 128), bh);
                }
            }
            wg::commit();
            wg::wait<1>();
            if (prev >= 0) { __syncwarp(); if (lane == 0) tc::mbar_arrive(&bar_empty[prev]); }
            prev = s;
            if (++s == NS) { s = 0; par ^= 1u; }
        }
        wg::wait_all();
        if (prev >= 0) { __syncwarp(); if (lane == 0) tc::mbar_arrive(&bar_empty[prev]); }
        asm volatile("bar.sync 8, 256;" ::: "memory");   // both halves are done reading the ring before either overwrites it
        // every stage has been consumed: park the accumulator over the ring, row-major [128][ACC_LD]
        {
            const int r0 = m * 64 + ((warp - NWORK) & 3) * 16 + (lane >> 2), c0 = (lane & 3) * 2;
#pragma unroll
            for (int jj = 0; jj < MMA_N / 8; ++jj) {
                float* d = accs + (size_t)r0 * ACC_LD + jj * 8 + c0;
                *reinterpret_cast<float2*>(d) = make_float2(acc[4 * jj], acc[4 * jj + 1]);
                *reinterpret_cast<float2*>(d + 8 * ACC_LD) = make_float2(acc[4 * jj + 2], acc[4 * jj + 3]);
            }
            tc::mbar_arrive(&bar_acc);
        }
    } else {
        // =============================================================================== WORKERS
        const int wi = warp;
        const int q = warp & 3;
        const int row = q * 32 + lane;                // the tile row of this thread's epilogue
        const bool row_ok = row < rows;
        const int grow = row0 + (row_ok ? row : 0);
        constexpr int NCG = NWORK / 4;                // epilogue column groups
        const int cgp = wi >> 2;
        const int nchunks = NC >> 3;
        bool ok = true;
        const int NKC = DP >> 3;
        if (GATHER) {
            const int grp = wi >> 2;
            const int gi = (wi & 3) * 32 + lane;      // the tile row this thread gathers
            // ---- the tile's (target, type) -> source table
            for (int i = tid; i < TILE_M * T; i += NWORK * 32) sPair[i] = p.pair_src[(size_t)row0 * T + i];
            // ---- virtual rows: the pairs of this tile with several messages, summed in message order (fp32), re-split, stored as image rows,
            // for every K group before the first stage is gathered
            const int v0 = p.tile_vptr[tile], nv = p.tile_vptr[tile + 1] - v0;
            for (int jg = 0; jg < GPS; ++jg) {
                const int ks0 = jg * KS, nks = min(KS, NKS - ks0);
                for (int task = tid; task < nv * nks; task += NWORK * 32) {
                    const int vl = task / nks, vid = v0 + vl, ks = ks0 + (task - vl * nks);
                    const int4 i0 = __ldg(p.vinfo + 2 * (size_t)vid), i1 = __ldg(p.vinfo + 2 * (size_t)vid + 1);
                    uint4 h0, l0, h1, l1;
                    if (p.slot_w)
                        sum_pair_sources_weighted(p.g_img, NKS, ks, i0, i1, p.vsrc + p.vrow_ptr[i0.x > 7 ? vid : 0], p.slot_w + p.vslot[vid], h0, h1,
                                                  l0, l1);
                    else
                        sum_pair_sources(p.g_img, NKS, ks, i0, i1, p.vsrc + p.vrow_ptr[i0.x > 7 ? vid : 0], h0, h1, l0, l1);
                    uint8_t* vp = p.virt_img + ((size_t)(vid >> 7) * NKS + ks) * A_STAGE_B + (size_t)(vid & 127) * 16;
                    *reinterpret_cast<uint4*>(vp) = h0;
                    *reinterpret_cast<uint4*>(vp + 2048) = h1;
                    *reinterpret_cast<uint4*>(vp + 4096) = l0;
                    *reinterpret_cast<uint4*>(vp + 6144) = l1;
                }
            }
            __threadfence();   // the copies below read these rows back through L2 (cp.async.cg)
            asm volatile("bar.sync 1, %0;" ::"n"(NWORK * 32) : "memory");
            // group `grp` fills stages grp, grp + NGATHER, ...: every row is an asynchronous 64-byte copy per K-step (or zeros).
            // The ring has at least NGATHER stages (MIN_NS), so the parity waits below are sound.
            for (int g = grp; g < ng && ok; g += NGATHER) {
                const int j = g / nsegs, sg = g - j * nsegs;   // K group major: stage g = (K group j, present edge type sg)
                const int s = g % NS, round = g / NS;
                const int ks0 = j * KS, nks = min(KS, NKS - ks0);
                const int ps = sPair[gi * T + s_types[sg]];
                const uint8_t* sp = nullptr;
                if (ps >= 0) sp = p.g_img + ((size_t)(ps >> 7) * NKS + ks0) * A_STAGE_B + (size_t)(ps & 127) * 16;
                else if (ps < -1) { const int vid = -(ps + 2); sp = p.virt_img + ((size_t)(vid >> 7) * NKS + ks0) * A_STAGE_B + (size_t)(vid & 127) * 16; }
                // one warp of the group polls the stage's barrier, the other three block on a hardware barrier (polling warps cost issue slots)
                if (round > 0 && (wi & 3) == 0 && !tc::mbar_wait(&bar_empty[s], (uint32_t)(round - 1) & 1u, abortp)) *abortp = 1;
                asm volatile("bar.sync %0, 128;" ::"r"(2 + grp) : "memory");
                if (*abortp) { ok = false; break; }
                uint8_t* ap = smem + (size_t)s * STAGE_B + (size_t)gi * 16;
                const uint32_t bar = smem_u32(&bar_afull[s]);
                if (sp) {
                    uint32_t dst = smem_u32(ap);
                    for (int i = 0; i < nks; ++i, dst += A_STAGE_B, sp += A_STAGE_B) {
                        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(sp) : "memory");
                        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst + 2048u), "l"(sp + 2048) : "memory");
                        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst + 4096u), "l"(sp + 4096) : "memory");
                        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst + 6144u), "l"(sp + 6144) : "memory");
                    }
                    // one arrival on the stage's barrier when this thread's copies have landed (the barrier counts 128 threads)
                    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(bar) : "memory");
                } else {
                    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
                    for (int i = 0; i < nks; ++i, ap += A_STAGE_B) {
                        *reinterpret_cast<uint4*>(ap) = z;
                        *reinterpret_cast<uint4*>(ap + 2048) = z;
                        *reinterpret_cast<uint4*>(ap + 4096) = z;
                        *reinterpret_cast<uint4*>(ap + 6144) = z;
                    }
                    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
                }
            }
        }
        // ---- epilogue: parked accumulator -> registers -> outputs.  The global operands of the first chunk are requested BEFORE the wait for the
        // accumulator, those of chunk c+1 before the math of chunk c (the loads are L2 hits after the prefetch above).
        const bool have_acc = nk > 0;
        // the cells: GRU and CudnnCompatibleGRUCell have gates (u blends the candidate with h), CudnnCompatibleGRUCell resets after the
        // recurrent product, RNN has neither
        const bool gated = p.cell != CELL_RNN, cudnn = p.cell == CELL_CUDNN_GRU;
        const int colb = nb0 * NC;                    // first (padded) output column of this CTA
        const float* acc_row = accs + (size_t)row * ACC_LD;
        // the global operands of this thread's next chunk are requested before the math of the current one
        float hA[8], uA[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { hA[j] = 0.0f; uA[j] = 0.0f; }
        const bool cand_h = p.epi == EPI_CAND && (gated || p.sv_h);
        auto load_ops = [&](int c, float (&hb)[8], float (&ub)[8]) {   // operands of chunk c (if it exists)
            const int colp = colb + c * 8;
            if (c >= nchunks) return;
            if (p.epi == EPI_CAND) {
                if (colp >= DP) return;
                if (cand_h) chunk_load(p.h_chk, NKC, tile, colp >> 3, row, hb);
                if (gated) chunk_load(p.u_buf, NKC, tile, colp >> 3, row, ub);
            } else if (p.epi == EPI_GATE) {
                if (colp < DP) chunk_load(p.h_chk, NKC, tile, colp >> 3, row, hb);
            } else if (p.epi == EPI_HPROJ) {
                if (colp < DP) chunk_load(p.rq_chk, NKC, tile, colp >> 3, row, hb);   // r
            }
        };
        if (!GATHER) load_ops(cgp, hA, uA);
        if (nk > 0) {   // worker warp 0 polls for the accumulator, the others block on the hardware barrier behind it
            if (wi == 0 && ok && !tc::mbar_wait(&bar_acc, 0, abortp)) *abortp = 1;
            asm volatile("bar.sync 1, %0;" ::"n"(NWORK * 32) : "memory");
            if (*abortp) ok = false;
        }
        if (ok) {
            if (p.epi == EPI_AGG) {
                // sparse:207-209 divides by (sum of in-degrees + 1e-7); one IEEE reciprocal per row, then a multiply per element (differs from
                // the quotient by at most 1 ulp; tests/test_gpu_stream.py bounds the growth over 32 timesteps)
                const float inv_den = (p.use_avg && row_ok) ? __frcp_rn(p.denom[grow]) : 1.0f;
                for (int c = cgp; c < nchunks; c += NCG) {
                    const int col = colb + c * 8;
                    if (col >= DP) break;
                    float v[8];
                    if (have_acc) tc::lds8(acc_row + c * 8, v);
                    else {
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] = 0.0f;
                    }
                    if (p.use_bias && row_ok) {
                        for (int t = 0; t < T; ++t) {
                            const float ind = p.indeg[(size_t)grow * T + t];
                            float b[8];
                            tc::load8_guarded(p.bias + (size_t)t * D, col, D, b);
#pragma unroll
                            for (int j = 0; j < 8; ++j) v[j] = fmaf(ind, b[j], v[j]);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] = row_ok ? v[j] * inv_den : 0.0f;
                    if (p.sv_agg && row_ok) tc::store8_guarded(p.sv_agg + (size_t)grow * D, col, D, v);
                    img_store_chunk(p.img_out, NKS, tile, row, col, v);
                }
            } else if (p.epi == EPI_GATE) {
                auto gate_chunk = [&](int c, float (&hb)[8], float (&ub)[8]) -> bool {
                    const int colp = colb + c * 8;
                    if (c >= nchunks || colp >= 2 * DP) return false;
                    const bool is_r = colp < DP;
                    const int col = is_r ? colp : colp - DP;
                    float g[8], b[8], h[8];
                    tc::lds8(acc_row + c * 8, g);
#pragma unroll
                    for (int j = 0; j < 8; ++j) h[j] = hb[j];
                    load_ops(c + NCG, hb, ub);
                    tc::load8_guarded(p.bias + (is_r ? 0 : D), col, D, b);
#pragma unroll
                    for (int j = 0; j < 8; ++j) g[j] = tc::sigmoid_fast(g[j] + b[j]);
                    if (is_r) {
                        if (p.sv_r && row_ok) {
                            tc::store8_guarded(p.sv_r + (size_t)grow * D, col, D, g);
                            tc::store8_guarded(p.sv_h + (size_t)grow * D, col, D, h);
                        }
                        if (cudnn) {   // r itself: the hidden-projection launch multiplies it by q
                            chunk_store(p.rq_chk, NKC, tile, col >> 3, row, g);
                        } else {
                            float rh[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j) rh[j] = g[j] * h[j];
                            img_store_chunk(p.img_out, NKS, tile, row, col, rh);
                        }
                    } else {
                        chunk_store(p.u_buf, NKC, tile, col >> 3, row, g);
                        if (p.sv_u && row_ok) tc::store8_guarded(p.sv_u + (size_t)grow * D, col, D, g);
                    }
                    return true;
                };
                for (int c = cgp; c < nchunks; c += NCG)
                    if (!gate_chunk(c, hA, uA)) break;
            } else if (p.epi == EPI_GCN) {
                // GCN layer: the arithmetic and the dropout mask of gcn::epilogue (ggnn_gcn.cuh); only the D real columns are written
                for (int c = cgp; c < nchunks && row_ok; c += NCG) {
                    const int col = colb + c * 8;
                    if (col >= D) break;
                    float v[8];
                    tc::lds8(acc_row + c * 8, v);
                    if (p.bias) {
                        float b[8];
                        tc::load8_guarded(p.bias, col, D, b);
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] += b[j];
                    }
                    if (p.relu_dropout) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            v[j] = fmaxf(v[j], 0.0f);
                            if (p.drop_keep < 1.0f) v[j] = dropout_apply(v[j], p.drop_seed, p.gstep, p.V, D, grow, col + j, p.drop_keep);
                        }
                    }
                    tc::store8_guarded(p.h_out + (size_t)grow * D, col, D, v);
                }
            } else if (p.epi == EPI_HPROJ) {
                // CudnnCompatibleGRUCell: q = h . K_hid + b_hid (saved for the backward pass), and the r chunk becomes r*q
                auto hproj_chunk = [&](int c, float (&hb)[8], float (&ub)[8]) -> bool {
                    const int col = colb + c * 8;
                    if (c >= nchunks || col >= DP) return false;
                    float q[8], b[8], r[8];
                    tc::lds8(acc_row + c * 8, q);
#pragma unroll
                    for (int j = 0; j < 8; ++j) r[j] = hb[j];
                    load_ops(c + NCG, hb, ub);
                    tc::load8_guarded(p.b_hid, col, D, b);
#pragma unroll
                    for (int j = 0; j < 8; ++j) { q[j] += b[j]; r[j] *= q[j]; }
                    if (p.sv_q && row_ok) tc::store8_guarded(p.sv_q + (size_t)grow * D, col, D, q);
                    chunk_store(p.rq_chk, NKC, tile, col >> 3, row, r);
                    return true;
                };
                for (int c = cgp; c < nchunks; c += NCG)
                    if (!hproj_chunk(c, hA, uA)) break;
            } else {
                auto cand_chunk = [&](int c, float (&hb)[8], float (&ub)[8]) -> bool {
                    const int col = colb + c * 8;
                    if (c >= nchunks || col >= DP) return false;
                    float cv[8], b[8], h[8], u[8], hn[8];
                    tc::lds8(acc_row + c * 8, cv);
#pragma unroll
                    for (int j = 0; j < 8; ++j) { h[j] = hb[j]; u[j] = ub[j]; }
                    load_ops(c + NCG, hb, ub);
                    tc::load8_guarded(p.bias, col, D, b);
                    if (gated) {
                        if (cudnn) {   // c = tanh(x . K_in + b_in + r*q), r*q from the hidden-projection launch
                            float rq[8];
                            chunk_load(p.rq_chk, NKC, tile, col >> 3, row, rq);
#pragma unroll
                            for (int j = 0; j < 8; ++j) cv[j] = tc::act_fast(cv[j] + b[j] + rq[j], p.act);
                        } else {
#pragma unroll
                            for (int j = 0; j < 8; ++j) cv[j] = tc::act_fast(cv[j] + b[j], p.act);
                        }
#pragma unroll
                        for (int j = 0; j < 8; ++j) hn[j] = fmaf(u[j], h[j] - cv[j], cv[j]);   // u*h + (1-u)*c
                        if (p.sv_c && row_ok) tc::store8_guarded(p.sv_c + (size_t)grow * D, col, D, cv);
                    } else {
#pragma unroll
                        for (int j = 0; j < 8; ++j) hn[j] = tc::act_fast(cv[j] + b[j], p.act);
                        if (p.sv_h && row_ok) tc::store8_guarded(p.sv_h + (size_t)grow * D, col, D, h);
                    }
                    if (p.drop_keep < 1.0f) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) hn[j] = dropout_apply(hn[j], p.drop_seed, p.gstep, p.V, D, grow, col + j, p.drop_keep);
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) hn[j] = (row_ok && col + j < D) ? hn[j] : 0.0f;
                    chunk_store(p.h_chk_out, NKC, tile, col >> 3, row, hn);
                    if (p.h_out && row_ok) tc::store8_guarded(p.h_out + (size_t)grow * D, col, D, hn);
                    img_store_chunk(p.img_out, NKS, tile, row, col, hn);
                    return true;
                };
                for (int c = cgp; c < nchunks; c += NCG)
                    if (!cand_chunk(c, hA, uA)) break;
            }
        }
        if (!ok && lane == 0) atomicExch(p.error_flag, 11);
    }
    __syncthreads();
}

// Propagation attention (sparse:170-196) on the streaming plan: the pre-pass of a timestep, before its gather launch.  The arithmetic of
// step::attention_kernel (one warp per target node, fp32 scores <h[src], h[v]> * a_t, max-shifted expf, sum + 1e-7, a division), read
// from the chunk-major fp32 master `chk` of the step's input state -- never from the bf16 images, whose split error times a score of
// order 100 would move the probabilities far off -- and only over the D real columns.  att[slot] = the probability of each target-CSR
// slot, which the gather launch reads as its slot weights.  No atomics.
__global__ void __launch_bounds__(256) attention_chunk_kernel(const int* __restrict__ row_ptr, const int* __restrict__ csr_src,
                                                              const float* __restrict__ chk, const float* __restrict__ att_w,
                                                              float* __restrict__ att, int V, int D, int DP, int T) {
    const int v = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (v >= V) return;
    const int D4 = D >> 2, NKC = DP >> 3;
    const float* hv = chk + chunk_off(NKC, v >> 7, 0, v & 127);
    const int mbeg = row_ptr[(size_t)v * T], mend = row_ptr[(size_t)(v + 1) * T];
    float mx = -INFINITY;
    for (int t = 0; t < T; ++t) {
        const float aw = att_w[t];
        const int beg = row_ptr[(size_t)v * T + t], end = row_ptr[(size_t)v * T + t + 1];
        for (int m = beg; m < end; ++m) {
            const int src = csr_src[m];
            const float* hp = chk + chunk_off(NKC, src >> 7, 0, src & 127);
            float dot = 0.f;
            for (int c4 = lane; c4 < D4; c4 += 32) {   // columns 4*c4 .. 4*c4+3: half c4 & 1 of chunk c4 / 2, 128 rows x 8 floats apart
                const size_t o = (size_t)(c4 >> 1) * (TILE_M * 8) + (c4 & 1) * 4;
                const float4 a = *reinterpret_cast<const float4*>(hp + o), b = *reinterpret_cast<const float4*>(hv + o);
                dot += a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
            const float sc = dot * aw;
            if (lane == 0) att[m] = sc;
            mx = fmaxf(mx, sc);
        }
    }
    __syncwarp();
    float sum = 0.f;
    for (int m = mbeg + lane; m < mend; m += 32) {
        const float ex = expf(att[m] - mx);
        att[m] = ex;
        sum += ex;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float den = sum + 1e-7f;   // SMALL_NUMBER, sparse:194
    for (int m = mbeg + lane; m < mend; m += 32) att[m] = att[m] / den;
}

// fp32 [V][D] row-major -> tile-major bf16 hi/lo image + chunk-major fp32 copy ([ntiles*128][DP], zero padded)
__global__ void ggnn_image_kernel(const float* __restrict__ x, uint8_t* __restrict__ img, float* __restrict__ chk, int V, int D, int DP, int ntiles) {
    const int NKC = DP >> 3, NKS = DP >> 4;
    const long long total = (long long)ntiles * TILE_M * NKC;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        // consecutive threads = consecutive rows of one chunk column: coalesced image writes
        const int row = (int)(idx % TILE_M);
        const int kc = (int)((idx / TILE_M) % NKC);
        const int tile = (int)(idx / ((long long)TILE_M * NKC));
        const int grow = tile * TILE_M + row;
        float v[8];
        tc::load8_guarded(x + (size_t)(grow < V ? grow : 0) * D, kc * 8, grow < V ? D : 0, v);
        img_store_chunk(img, NKS, tile, row, kc * 8, v);
        chunk_store(chk, NKC, tile, kc, row, v);
    }
}

// Weight pre-tiling for the streaming kernel.  Source: fp32 row-major W[(nseg*D) rows][src_ld cols]; the padded operand has
// K = nseg*DP rows (segment s, row kk < D -> source row s*D + kk) and N = nblk*NC columns, where padded column n maps to source
// column (n / DP)*D + n % DP when n % DP < D and n / DP < ncolblk (the [r | u] gate kernel has two D-wide column blocks), else zero.
//   out: [nblk][K/16] stages of 64*NC bytes:  byte(part, kg, n, j) = part*32*NC + kg*16*NC + n*16 + j*2
__global__ void ggnn_tile_weights_stream_kernel(const float* __restrict__ W, uint8_t* __restrict__ out, int D, int DP, int nseg, int ncolblk,
                                                int src_ld, int NC, int nblk) {
    const int kt = nseg * DP / 16;
    const long long total = (long long)nblk * kt * 2 * NC;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(idx % NC);
        const int kg = (int)((idx / NC) % 2);
        const int k = (int)((idx / (2 * NC)) % kt);
        const int nb = (int)(idx / ((long long)2 * NC * kt));
        const int np = nb * NC + n;
        const int cb = np / DP, nn = np - cb * DP;
        const bool col_ok = cb < ncolblk && nn < D;
        float x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int kp = k * 16 + kg * 8 + j;
            const int sg = kp / DP, kk = kp - sg * DP;
            x[j] = (col_ok && kk < D) ? W[(size_t)(sg * D + kk) * src_ld + cb * D + nn] : 0.0f;
        }
        uint4 hi, lo;
        tc::split8(x, hi, lo);
        uint8_t* base = out + ((size_t)nb * kt + k) * 64 * NC + (size_t)kg * 16 * NC + (size_t)n * 16;
        *reinterpret_cast<uint4*>(base) = hi;
        *reinterpret_cast<uint4*>(base + (size_t)32 * NC) = lo;
    }
}

}  // namespace ts
}  // namespace ggnn
