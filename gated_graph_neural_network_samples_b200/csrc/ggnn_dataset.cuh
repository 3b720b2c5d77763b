// Batch assembly from a device-resident dataset (ggnn_set_graph_dataset): the graph image of a batch of whole graphs, written on the device
// in exactly the layout the host builder uploads, plus h0, the targets and the readout map.
//
// Graphs never share edges, so every section of a batch's image is the graphs' own pieces laid end to end with offsets: a graph's
// target-CSR rows get the slots of earlier graphs added, its sources the node offset, its message ids the batch's type base plus the
// type's messages in earlier graphs; the source-keyed CSR, the attention slot map, the slot weights and the streaming tables (virtual row
// ids offset by the earlier graphs' virtual rows, their first slots by the earlier graphs' slots) the same.  The dataset holds each graph's pieces in graph-local numbering; the host half
// (ggnn_dataset_prepare_batch) computes the per-graph offsets, one record per graph of the batch.
//
// ds_graph_kernel: one block per graph of the batch, each writes its graph's rows, slots, nodes and labels -- no two blocks write the same
// byte, so there are no atomics and the image is a function of the dataset and the id list.  ds_tile_kernel then fills what depends on
// the tiles (tile starts, edge-type masks, first virtual row per tile) and the pair-table rows beyond the last node.
//
// A dense batch (ggnn_dataset_prepare_batch_dense, DsOut::v > 0) gives graph i the rows i*v .. i*v+v-1: the graph's own V_g rows, then
// v - V_g isolated padding rows, written as the host builder writes a row without messages (row_ptr = the graph's slot end, in-degree 0,
// denominator 0 + 1e-7, no source, h0 zero, node mask 0).  Sparse and GCN batches (v = 0) skip every padding branch.
#pragma once
#include "ggnn_common.cuh"
#include "ggnn_fwd_stream.cuh"

namespace ggnn {
namespace ds {

// A record of the batch table: the graph's dataset id and its offsets in the batch, then its message base per edge type.
enum { R_GID = 0, R_NODE = 1, R_SLOT = 2, R_VROW = 3, R_VSRC = 4, R_MBASE = 5 };
// A row of the dataset's per-graph table: where the graph's pieces start in the dataset arrays (N + 1 rows).
enum { B_NODE = 0, B_SLOT = 1, B_VROW = 2, B_VSRC = 3, B_WIDTH = 4 };

// The dataset's arrays (device, graph-local numbering, graphs in dataset order).  Absent arrays are null.
struct DsArrays {
    const int* base;       // [N+1][B_WIDTH]
    const int* row_end;    // [sum V*T] end of every (target, type) row within the graph's slots
    const int* src;        // [sum M] source node of every target-CSR slot
    const int* pos;        // [sum M] the slot's message position within its edge type's list of the graph
    const float* indeg;    // [sum V*T]
    const float* denom;    // [sum V]
    const int* trow_end;   // [sum V*T] source-keyed CSR (training datasets)
    const int* ttgt;       // [sum M]
    const int* tslot;      // [sum M] attention only: target-CSR slot of every source-keyed entry
    const int* pair;       // [sum V*T] streaming: -1, the one source, or -(2 + graph-local virtual row)
    const int* vend;       // [sum nv] end of every virtual row within the graph's virtual-row sources
    const int* vsrc;       // [sum nvm]
    const int* vpre;       // [sum V] virtual rows of the graph before every node
    const int* vslot;      // [sum nv] attention on the streaming plan: the first target-CSR slot of every virtual row within the graph's slots
    const float* slotw;    // [sum M] weighted (GCN): weight of every target-CSR slot
    const float* tslotw;   // [sum M] ... and of every source-keyed entry (training)
    const float* ann;      // [sum V][ann_size]
    const float* labels;   // [N][tasks]
    const float* lmask;    // [N][tasks]
    const int* nfeat;      // [N] dense datasets: the graph's feature count (its node mask is local row < nfeat)
    int ann_size, tasks;
};

// The batch's outputs: the sections of the graph image (null when the plan has none) and the caller's / the readout's buffers.
struct DsOut {
    ImageView img;
    float* h0;               // [V][D]
    float *tv, *tm;          // [tasks][G]
    int *ro_graph_of, *ro_start;
    float *node_mask, *ro_mask;       // dense batches: [V] the caller's node mask and the readout's copy
    int V, D, T, G, ntiles, nv, rec;   // rec: ints per batch record (R_MBASE + T)
    int v;                             // dense batches: rows per graph (nodes_per_graph); 0 for sparse and GCN batches
};

__global__ void __launch_bounds__(256) ds_graph_kernel(const DsArrays a, const DsOut o, const int* __restrict__ table) {
    const int i = blockIdx.x;
    const int* r = table + (size_t)i * o.rec;
    const int gid = r[R_GID], noff = r[R_NODE], soff = r[R_SLOT], voff = r[R_VROW], vsoff = r[R_VSRC];
    const int* b = a.base + (size_t)gid * B_WIDTH;
    const int nb = b[B_NODE], sb = b[B_SLOT], vb = b[B_VROW], vsb = b[B_VSRC];
    const int Vg = b[B_WIDTH + B_NODE] - nb, nvg = b[B_WIDTH + B_VROW] - vb;
    const int T = o.T;
    for (int k = threadIdx.x; k < Vg * T; k += blockDim.x) {
        const size_t dk = (size_t)nb * T + k, R = (size_t)noff * T + k;
        const int lo = k ? a.row_end[dk - 1] : 0, hi = a.row_end[dk];
        const int mb = r[R_MBASE + k % T];
        o.img.row_ptr[R + 1] = soff + hi;
        for (int m = lo; m < hi; ++m) {
            o.img.src[soff + m] = a.src[sb + m] + noff;
            o.img.msg[soff + m] = mb + a.pos[sb + m];
            if (o.img.slotw) o.img.slotw[soff + m] = a.slotw[sb + m];
        }
        o.img.indeg[R] = a.indeg[dk];
        if (o.img.trow) {
            const int tlo = k ? a.trow_end[dk - 1] : 0, thi = a.trow_end[dk];
            o.img.trow[R + 1] = soff + thi;
            for (int m = tlo; m < thi; ++m) {
                o.img.ttgt[soff + m] = a.ttgt[sb + m] + noff;
                if (o.img.tslot) o.img.tslot[soff + m] = a.tslot[sb + m] + soff;
                if (o.img.tslotw) o.img.tslotw[soff + m] = a.tslotw[sb + m];
            }
        }
        if (o.img.pair) {
            const int p = a.pair[dk];
            o.img.pair[R] = p == -1 ? -1 : (p >= 0 ? p + noff : p - voff);   // -(2 + vid) - voff = -(2 + vid + voff)
        }
    }
    if (o.img.pair)
        for (int j = threadIdx.x; j < nvg; j += blockDim.x) {
            const int lo = j ? a.vend[vb + j - 1] : 0, hi = a.vend[vb + j], cnt = hi - lo, vid = voff + j;
            o.img.vptr[vid + 1] = vsoff + hi;
            if (o.img.vslot) o.img.vslot[vid] = a.vslot[vb + j] + soff;   // a graph's (node, type) rows are contiguous: its slots are too
            o.img.vinfo[8 * vid] = cnt;
            for (int m = 0; m < 7; ++m) o.img.vinfo[8 * vid + 1 + m] = m < cnt ? a.vsrc[vsb + lo + m] + noff : 0;
            for (int m = 0; m < cnt; ++m) o.img.vsrc[vsoff + lo + m] = a.vsrc[vsb + lo + m] + noff;
        }
    for (int v = threadIdx.x; v < Vg; v += blockDim.x) {
        o.img.denom[noff + v] = a.denom[nb + v];
        o.ro_graph_of[noff + v] = i;
    }
    const int D = o.D, A = a.ann_size;
    for (size_t k = threadIdx.x; k < (size_t)Vg * D; k += blockDim.x) {
        const int v = (int)(k / D), c = (int)(k % D);
        o.h0[(size_t)noff * D + k] = c < A ? a.ann[(size_t)(nb + v) * A + c] : 0.0f;
    }
    if (o.v > 0) {   // dense: the node mask of the real rows, then the padding rows Vg .. v-1 (isolated, every slot pointer at the graph's end)
        const int nf = a.nfeat[gid], Mg = a.base[(size_t)(gid + 1) * B_WIDTH + B_SLOT] - sb, npad = o.v - Vg;
        for (int v = threadIdx.x; v < Vg; v += blockDim.x) {
            const float m = v < nf ? 1.0f : 0.0f;
            o.node_mask[noff + v] = m; o.ro_mask[noff + v] = m;
        }
        for (int k = threadIdx.x; k < npad * T; k += blockDim.x) {
            const size_t R = (size_t)(noff + Vg) * T + k;
            o.img.row_ptr[R + 1] = soff + Mg;
            o.img.indeg[R] = 0.0f;
            if (o.img.trow) o.img.trow[R + 1] = soff + Mg;
            if (o.img.pair) o.img.pair[R] = -1;
        }
        for (int v = Vg + threadIdx.x; v < o.v; v += blockDim.x) {
            o.img.denom[noff + v] = 0.0f + 1e-7f;
            o.ro_graph_of[noff + v] = i;
            o.node_mask[noff + v] = 0.0f; o.ro_mask[noff + v] = 0.0f;
        }
        for (size_t k = threadIdx.x; k < (size_t)npad * D; k += blockDim.x) o.h0[(size_t)(noff + Vg) * D + k] = 0.0f;
    }
    for (int t = threadIdx.x; t < a.tasks; t += blockDim.x) {
        o.tv[(size_t)t * o.G + i] = a.labels[(size_t)gid * a.tasks + t];
        o.tm[(size_t)t * o.G + i] = a.lmask[(size_t)gid * a.tasks + t];
    }
    if (threadIdx.x == 0) {
        o.ro_start[i] = noff;
        if (i == o.G - 1) o.ro_start[o.G] = o.V;
    }
}

// After ds_graph_kernel (it reads the batch's row_ptr): tiles, their edge-type masks, the first virtual row of every tile, and -1 in the
// pair-table rows of the last tile beyond V.  `tiles`: the plan's tile starts [ntiles + 1], uploaded with the batch table.
__global__ void __launch_bounds__(256) ds_tile_kernel(const DsArrays a, const DsOut o, const int* __restrict__ table, const int* __restrict__ tiles) {
    const int T = o.T;
    const size_t stride = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (size_t i = tid; i <= (size_t)o.ntiles; i += stride) {
        const int n = tiles[i];
        o.img.tile_start[i] = n;
        if (i < (size_t)o.ntiles) {
            unsigned mask = 0;
            for (size_t k = (size_t)n * T, kend = (size_t)tiles[i + 1] * T; k < kend; ++k) mask |= (unsigned)(o.img.row_ptr[k + 1] > o.img.row_ptr[k]) << (k % T);
            o.img.tile_mask[i] = mask;
        }
        if (o.img.pair) {   // virtual rows before node n: those of the graph holding n (the last graph starting at or before n) before it
            int v = o.nv;
            if (n < o.V) {
                int lo = 0, hi = o.G - 1;
                while (lo < hi) {
                    const int mid = (lo + hi + 1) / 2;
                    if (table[(size_t)mid * o.rec + R_NODE] <= n) lo = mid; else hi = mid - 1;
                }
                const int* r = table + (size_t)lo * o.rec;
                const int* gb = a.base + (size_t)r[R_GID] * B_WIDTH;
                const int local = n - r[R_NODE];
                if (o.v > 0 && local >= gb[B_WIDTH + B_NODE] - gb[B_NODE])   // dense: a tile starting in the graph's padding rows
                    v = r[R_VROW] + (gb[B_WIDTH + B_VROW] - gb[B_VROW]);
                else
                    v = r[R_VROW] + a.vpre[gb[B_NODE] + local];
            }
            o.img.tvp[i] = v;
        }
    }
    if (o.img.pair)
        for (size_t k = (size_t)o.V * T + tid, kend = (size_t)max(o.ntiles, 1) * ts::TILE_M * T; k < kend; k += stride) o.img.pair[k] = -1;
}

}  // namespace ds
}  // namespace ggnn
