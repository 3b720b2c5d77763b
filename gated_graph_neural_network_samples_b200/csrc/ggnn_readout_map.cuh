// The readout map from DEVICE arrays (ggnn_readout_set_graphs_device): the sections ggnn_readout_set_graphs builds on the host --
// graph_of [V] | start [G+1] | mask [V] | perm [V] of readout_layout -- written by kernels into the engine's ro_buf.
//
// Determinism: atomics only count (the per-graph node counts, the first bad node as a minimum, the ungrouped flag), and each such result
// is the same whatever order the atomics land in.  start is CUB's exclusive scan of the counts and perm CUB's stable radix sort of the
// node indices keyed by graph, the host's stable counting sort; every other section has one writer per element.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace ggnn {
namespace ro_map {

// The summary read back after the map pass.  BAD: the lowest out-of-range node (0xffffffff: none); UNGROUPED: 1 when some node's graph
// is below its predecessor's.
enum { S_BAD = 0, S_UNGROUPED, S_COUNT };

// One thread per node v of the caller's graph_nodes_list: validate 0 <= g < G (a bad node lowers the first-bad minimum and writes
// nothing else), write graph_of[v], count v into its graph, and raise the ungrouped flag when g < gnl[v-1].  On the success path every
// entry is in range, so comparing with the raw predecessor is the host's comparison with graph_of[v-1].
__global__ void __launch_bounds__(256) graph_map_kernel(const int32_t* __restrict__ gnl, int V, int G, int* __restrict__ graph_of,
                                                        int* __restrict__ counts, unsigned* __restrict__ summary) {
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
        const int g = gnl[v];
        if ((unsigned)g >= (unsigned)G) {
            atomicMin(summary + S_BAD, (unsigned)v);
            continue;
        }
        graph_of[v] = g;
        atomicAdd(counts + g, 1);
        if (v > 0 && g < gnl[v - 1]) summary[S_UNGROUPED] = 1u;   // every writer stores the same value
    }
}

// The node indices 0 .. V-1: the values CUB's sort carries into perm.
__global__ void __launch_bounds__(256) node_ids_kernel(int V, int* __restrict__ ids) {
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) ids[v] = v;
}

// The dense map (no list, V = G * npg): graph_of[r] = r / npg for r < V and start[g] = g * npg for g <= G.
__global__ void __launch_bounds__(256) dense_map_kernel(int V, int G, int npg, int* __restrict__ graph_of, int* __restrict__ start) {
    const int64_t n = V > G ? (int64_t)V : (int64_t)G + 1;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < V) graph_of[i] = (int)i / npg;
        if (i <= G) start[i] = (int)i * npg;   // <= V
    }
}

}  // namespace ro_map
}  // namespace ggnn
