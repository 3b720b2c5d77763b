// Sparse batches from DEVICE adjacency lists (ggnn_set_graph_sparse_device, and ggnn_set_graph_gcn_device after dg_gcn's pass): the section
// fills of build_sparse_image as kernels, writing the same image into the engine's graph buffer.  The plan and the layout stay on the host (build_plan, layout_image, image_view): these
// kernels only count, derive the cut points and totals the plan needs, and fill the sections the plan carries.
//
// Determinism: atomics only count (per-row message counts, reach maxima, the first bad edge as a minimum, the per-tile maxima), and every
// such result is the same whatever order the atomics land in.  Slots are placed by CUB's stable radix sort of the messages by row key, in
// the reference's type-major message order -- NumPy's stable argsort by (target, type), as the host builder's counting sort -- and every
// other section has one writer per element.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "ggnn_common.cuh"
#include "ggnn_fwd_stream.cuh"

namespace ggnn {
namespace dg {

constexpr int MAX_TYPES = 32;

// The caller's per-type lists: adj[t] -> [E_t][2] int32 (source, target); base[t] = the type's first message in the type-major order,
// base[T] = M.  Passed by value (T <= 32).
struct EdgeLists {
    const int32_t* adj[MAX_TYPES];
    int64_t base[MAX_TYPES + 1];
    int T;
};

// The summary read back after the counting passes.  BAD: the first out-of-range message (0xffffffff: none); NV2 / NVM2: (target, type)
// rows with >= 2 messages and their messages; NV1: rows with >= 1 message (the all-virtual count, whose messages are all M); NCUT: interior
// cut points.  BAD_T .. BAD_D: the first bad edge's type, index and values.
enum { S_BAD = 0, S_NV2, S_NVM2, S_NV1, S_NCUT, S_BAD_T, S_BAD_I, S_BAD_S, S_BAD_D, S_COUNT };

__device__ __forceinline__ int type_of(const EdgeLists& L, int64_t m) {
    int lo = 0, hi = L.T - 1;   // the last type whose base is <= m
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (L.base[mid] <= m) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Pass 1, one thread per message m (type-major order): validate; count the message into its target row d*T+t (and, for the source-keyed
// CSR, its source row s*T+t); raise reach[min(s,d)] to max(s,d); write the sort keys, the message id and the endpoints.  An out-of-range
// edge lowers the first-bad minimum and writes nothing else.
__global__ void __launch_bounds__(256) count_kernel(const EdgeLists L, int V, int64_t M, int* __restrict__ counts, int* __restrict__ tcounts,
                                                    int* __restrict__ reach, int* __restrict__ key, int* __restrict__ tkey, int* __restrict__ ids,
                                                    int* __restrict__ es, int* __restrict__ ed, unsigned* __restrict__ summary) {
    const int T = L.T;
    for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m < M; m += (int64_t)gridDim.x * blockDim.x) {
        const int t = type_of(L, m);
        const int64_t i = m - L.base[t];
        const int s = L.adj[t][2 * i], d = L.adj[t][2 * i + 1];
        if ((unsigned)s >= (unsigned)V || (unsigned)d >= (unsigned)V) {
            atomicMin(summary + S_BAD, (unsigned)m);
            continue;
        }
        atomicAdd(counts + ((size_t)d * T + t), 1);
        if (tcounts) atomicAdd(tcounts + ((size_t)s * T + t), 1);
        if (reach) atomicMax(reach + min(s, d), max(s, d));
        key[m] = d * T + t;
        if (tkey) tkey[m] = s * T + t;
        ids[m] = (int)m;
        es[m] = s; ed[m] = d;
    }
}

// The virtual-row totals over the V*T row counts (integer sums: the same in every order) and, from block 0, the first bad edge's values.
__global__ void __launch_bounds__(256) summary_kernel(const EdgeLists L, const int* __restrict__ counts, int64_t VT, unsigned* __restrict__ summary) {
    unsigned nv2 = 0, nvm2 = 0, nv1 = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < VT; r += (int64_t)gridDim.x * blockDim.x) {
        const int c = counts[r];
        nv1 += c >= 1;
        if (c >= 2) { ++nv2; nvm2 += c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        nv2 += __shfl_xor_sync(0xffffffffu, nv2, o);
        nvm2 += __shfl_xor_sync(0xffffffffu, nvm2, o);
        nv1 += __shfl_xor_sync(0xffffffffu, nv1, o);
    }
    if ((threadIdx.x & 31) == 0 && (nv2 | nv1)) {
        atomicAdd(summary + S_NV2, nv2); atomicAdd(summary + S_NVM2, nvm2); atomicAdd(summary + S_NV1, nv1);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && summary[S_BAD] != 0xffffffffu) {
        const int64_t m = summary[S_BAD];
        const int t = type_of(L, m);
        const int64_t i = m - L.base[t];
        summary[S_BAD_T] = (unsigned)t; summary[S_BAD_I] = (unsigned)i;
        summary[S_BAD_S] = (unsigned)L.adj[t][2 * i]; summary[S_BAD_D] = (unsigned)L.adj[t][2 * i + 1];
    }
}

// find_cuts' rule on the device: the boundary before node i (0 < i < V) is a cut point iff far[i-1] = max_{j < i} reach[j] < i.  flag[i-1]
// marks it; flag[V-1] = 0 closes the range for the exclusive scan that numbers the cut points.
__global__ void __launch_bounds__(256) cut_flags_kernel(const int* __restrict__ far, int V, int* __restrict__ flag) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x + 1; i <= V; i += gridDim.x * blockDim.x) flag[i - 1] = i < V && far[i - 1] < i;
}

// The cut points in ascending order (pos: the exclusive scan of the flags) and their number into the summary.
__global__ void __launch_bounds__(256) cut_list_kernel(const int* __restrict__ flag, const int* __restrict__ pos, int V, int* __restrict__ cuts,
                                                       unsigned* __restrict__ summary) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x + 1; i < V; i += gridDim.x * blockDim.x)
        if (flag[i - 1]) cuts[pos[i - 1]] = i;
    if (blockIdx.x == 0 && threadIdx.x == 0) summary[S_NCUT] = (unsigned)pos[V - 1];
}

// In-degrees from the row counts (the NULL table: per-(target, type) message counts as fp32) and the denominators of fill_denominators:
// the fp32 sum over the type axis in type order, + 1e-7.
__global__ void __launch_bounds__(256) indeg_kernel(const int* __restrict__ counts, int64_t VT, float* __restrict__ indeg) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < VT; r += (int64_t)gridDim.x * blockDim.x) indeg[r] = (float)counts[r];
}

__global__ void __launch_bounds__(256) denom_kernel(const float* __restrict__ indeg, int V, int T, float* __restrict__ denom) {
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
        const float* row = indeg + (size_t)v * T;
        float s = 0.0f;
        for (int t = 0; t < T; ++t) s += row[t];
        denom[v] = s + 1e-7f;
    }
}

// The target CSR's sources from its message ids (msg: the sorted ids), and with `slot_of` the inverse map message -> target slot.
__global__ void __launch_bounds__(256) csr_src_kernel(const int* __restrict__ msg, const int* __restrict__ es, int64_t M, int* __restrict__ src,
                                                      int* __restrict__ slot_of) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < M; k += (int64_t)gridDim.x * blockDim.x) {
        const int m = msg[k];
        src[k] = es[m];
        if (slot_of) slot_of[m] = (int)k;
    }
}

// The source-keyed CSR's targets and (with `tslot`) target slots, from its message ids sorted by source row.
__global__ void __launch_bounds__(256) source_csr_kernel(const int* __restrict__ tmsg, const int* __restrict__ ed, const int* __restrict__ slot_of,
                                                         int64_t M, int* __restrict__ ttgt, int* __restrict__ tslot) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < M; j += (int64_t)gridDim.x * blockDim.x) {
        const int m = tmsg[j];
        ttgt[j] = ed[m];
        if (tslot) tslot[j] = slot_of[m];
    }
}

// Streaming plan: which rows are virtual (several messages, or any message when `all_virtual`) and their message counts, for the two
// exclusive scans that number the virtual rows and place their sources.  Entry VT is 0.
__global__ void __launch_bounds__(256) virtual_flags_kernel(const int* __restrict__ counts, int64_t VT, bool all_virtual, int* __restrict__ vid,
                                                            int* __restrict__ vm) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= VT; r += (int64_t)gridDim.x * blockDim.x) {
        const int c = r < VT ? counts[r] : 0;
        const bool virt = c >= 2 || (all_virtual && c == 1);
        vid[r] = virt;
        vm[r] = virt ? c : 0;
    }
}

// stream_rows on the device, one thread per (target, type) row of the padded pair table (npairs = max(ntiles, 1) * TILE_M * T): -1 for no
// message and for rows beyond V, the one source, or -(2 + vid) for a virtual row, whose sources, end, first slot and vinfo record it writes
// (vid / vm: the exclusive scans of virtual_flags_kernel).
__global__ void __launch_bounds__(256) stream_rows_kernel(const int* __restrict__ row_ptr, const int* __restrict__ src, const int* __restrict__ vid,
                                                          const int* __restrict__ vm, int64_t VT, int64_t npairs, bool all_virtual,
                                                          int* __restrict__ pair, int* __restrict__ vptr, int* __restrict__ vsrc,
                                                          int* __restrict__ vinfo, int* __restrict__ vslot) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < npairs; r += (int64_t)gridDim.x * blockDim.x) {
        if (r >= VT) { pair[r] = -1; continue; }
        const int b = row_ptr[r], cnt = row_ptr[r + 1] - b;
        if (cnt == 0) { pair[r] = -1; continue; }
        if (cnt == 1 && !all_virtual) { pair[r] = src[b]; continue; }
        const int v = vid[r], at = vm[r];
        pair[r] = -(2 + v);
        if (vslot) vslot[v] = b;
        vinfo[8 * v] = cnt;
        for (int m = 0; m < 7; ++m) vinfo[8 * v + 1 + m] = m < cnt ? src[b + m] : 0;
        for (int m = 0; m < cnt; ++m) vsrc[at + m] = src[b + m];
        vptr[v + 1] = at + cnt;
    }
}

// The tile-dependent pass, one thread per tile start (ntiles + 1): the tile starts, every tile's edge-type mask and, into maxima[0] / [1],
// the largest message count and edge-type count of a tile; on the streaming plan the first virtual row of every tile (tvp, from the
// virtual-row scan, whose entry VT is the total).
__global__ void __launch_bounds__(256) tile_kernel(const int* __restrict__ tiles, int ntiles, int T, const int* __restrict__ row_ptr,
                                                   const int* __restrict__ vid, int* __restrict__ tile_start, unsigned* __restrict__ tile_mask,
                                                   int* __restrict__ tvp, int* __restrict__ maxima) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= ntiles; i += gridDim.x * blockDim.x) {
        const int n = tiles[i];
        tile_start[i] = n;
        if (tvp) tvp[i] = vid[(size_t)n * T];
        if (i == ntiles) continue;
        const size_t k0 = (size_t)n * T, k1 = (size_t)tiles[i + 1] * T;
        unsigned mask = 0;
        for (size_t k = k0; k < k1; ++k) mask |= (unsigned)(row_ptr[k + 1] > row_ptr[k]) << (k % T);
        tile_mask[i] = mask;
        atomicMax(maxima, row_ptr[k1] - row_ptr[k0]);
        atomicMax(maxima + 1, __popc(mask));
    }
}

}  // namespace dg

// The GCN entry's one pass ahead of dg's (ggnn_set_graph_gcn_device): gcn_pairs on the device.  It lives beside dg, which holds the passes
// both entries share.
namespace dg_gcn {

// One thread per entry k of the caller's [nnz, 2] int64 list (row i = output, column j = input): checks 0 <= i, j < V in int64 and writes
// the int32 pair (source j, target i) into `pairs`, the GCN's one edge type in list order.  An out-of-range entry lowers the first-bad
// minimum and writes (-1, -1), which count_kernel rejects, so nothing of it is counted.
__global__ void __launch_bounds__(256) gcn_pairs_kernel(const int64_t* __restrict__ list, int64_t nnz, int V, int32_t* __restrict__ pairs,
                                                        unsigned* __restrict__ summary) {
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = list[2 * k], j = list[2 * k + 1];   // two 8-byte loads: the ABI promises no more than int64 alignment
        const bool ok = (uint64_t)i < (uint64_t)V && (uint64_t)j < (uint64_t)V;
        if (!ok) atomicMin(summary + dg::S_BAD, (unsigned)k);
        reinterpret_cast<int2*>(pairs)[k] = ok ? make_int2((int)j, (int)i) : make_int2(-1, -1);
    }
}

}  // namespace dg_gcn
}  // namespace ggnn
