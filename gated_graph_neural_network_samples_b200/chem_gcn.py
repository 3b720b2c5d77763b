"""``SparseGCNChemModel`` with the reference's hook names, parameter keys and feed-dict slots (chem_tensorflow_gcn.py:28-199), its
propagation replaced by the H100 engine.

    prepare_specific_graph_model()        gcn:42-57   -> creates the trainables + the GCN engine handle
    compute_final_node_representations()  gcn:59-82   -> ggnn_set_graph_gcn (or a prepared graph, or ggnn_set_graph_gcn_device for a
                                                         CUDA feed) + ggnn_forward (C ABI)
    gated_regression()                    gcn:84-93   -> the sparse GGNN's readout (sparse:220-231 is the same graph)
"""
from __future__ import annotations

from typing import Any, Optional, Sequence

import numpy as np

from . import packing
from .chem_model import ChemModel
from .chem_sparse import SparseGGNNChemModel
from .engine import GCNEngine, GgnnError
from .readout import gated_readout_function
from .utils import glorot_init


def _propagation_function():
    import torch

    class GCNPropagation(torch.autograd.Function):
        """Autograd node around the C ABI: forward = ggnn_gcn_set_weights + ggnn_forward, backward = ggnn_gcn_backward.
        ``weights`` are the L kernels, then the L biases when the engine uses them, and, when they hold one more, the adjacency weights
        [num_messages()] of a message-weighted batch (set before the forward, their gradient from ggnn_gcn_backward_weighted)."""

        @staticmethod
        def forward(ctx, engine, h0, *weights):
            L = engine.L
            n_layer = L * (2 if engine.use_bias else 1)
            aw = weights[n_layer] if len(weights) > n_layer else None
            # ctx.needs_input_grad is all False under torch.no_grad() (validation epochs): no activations are saved there
            need = any(ctx.needs_input_grad[1:])
            kernels = [k.detach().contiguous() for k in weights[:L]]
            biases = [b.detach().contiguous() for b in weights[L:n_layer]] or None
            engine.set_weights(kernels, biases)
            if aw is not None:
                aw = aw.detach().contiguous()
                engine.set_message_weights(aw)
            engine.set_deterministic(torch.are_deterministic_algorithms_enabled())
            engine.set_save_for_backward(need)
            out = engine.forward(h0.detach().contiguous())
            ctx.aw_index = n_layer if aw is not None and ctx.needs_input_grad[2 + n_layer] else None
            ctx.serial = engine.serial   # the backward refuses once another forward, graph or weights replaced this one's
            ctx.engine, ctx.shapes = engine, [t.shape for t in weights]
            ctx.h0_needs = bool(ctx.needs_input_grad[1])
            ctx.keepalive = (h0, out, kernels, biases)   # the engine reads these buffers again in ggnn_gcn_backward
            return out

        @staticmethod
        def backward(ctx, d_out):
            ctx.engine.require_serial(ctx.serial, "the GCN propagation's backward")
            L = ctx.engine.L
            n_layer = L * (2 if ctx.engine.use_bias else 1)
            grads = [torch.zeros(s, dtype=torch.float32, device=d_out.device) for s in ctx.shapes]
            layers = [{'kernel': grads[l], 'bias': grads[L + l] if n_layer > L else None} for l in range(L)]
            d_h0 = torch.zeros_like(d_out) if ctx.h0_needs else None
            ctx.engine.set_deterministic(torch.are_deterministic_algorithms_enabled())
            if ctx.aw_index is None:
                ctx.engine.backward(d_out.contiguous(), layers, d_h0)
            else:
                ctx.engine.backward(d_out.contiguous(), layers, d_h0, d_adjacency_weights=grads[ctx.aw_index])
            return (None, d_h0) + tuple(grads)

    return GCNPropagation


def propagate(engine: GCNEngine, h0, kernels: Sequence, biases: Optional[Sequence] = None, adjacency_weights=None):
    """The sparse GCN propagation as a differentiable torch function, without a ChemModel: ``engine`` holds the current batch (for
    ``adjacency_weights``, a message-weighted one: ``prepare_graph_gcn_message_weighted`` + ``set_graph_prepared``, or, with the list on
    the GPU, the device-built batch of ``set_graph_gcn_device``), ``h0`` [V, D],
    ``kernels[l]`` [D, D] and, when the engine uses biases, ``biases[l]`` [D], fp32 CUDA tensors, and ``adjacency_weights`` an fp32 CUDA
    tensor [nnz] in list order (the weights of ``adjacency_weights`` in ``set_graph_gcn``, computed in torch: a learned or renormalized
    ``D^-1/2 (A+I) D^-1/2``, a DropEdge mask).  Returns the last layer's node states [V, D]; gradients reach ``h0``, every kernel and bias,
    and ``adjacency_weights``."""
    if (biases is not None) != engine.use_bias or len(kernels) != engine.L:
        raise GgnnError("expected %d kernels%s" % (engine.L, " and %d biases" % engine.L if engine.use_bias else " and no biases"))
    weights = list(kernels) + (list(biases) if biases is not None else [])
    if adjacency_weights is not None:
        weights.append(adjacency_weights)
    return _propagation_function().apply(engine, h0, *weights)


class SparseGCNChemModel(ChemModel):
    def __init__(self, args):
        super().__init__(args)

    @classmethod
    def default_params(cls):
        params = dict(super().default_params())
        params.update({  # gcn:33-40; the number of layers is the base key num_timesteps
            'batch_size': 100000,
            'task_sample_ratios': {},
            'gcn_use_bias': False,
            'graph_state_dropout_keep_prob': 1.0,
        })
        return params

    # ------------------------------------------------------------------ hook 1 (gcn:42-57)
    def prepare_specific_graph_model(self) -> None:
        import torch
        h_dim = self.params['hidden_size']
        for k in ('initial_node_representation', 'adjacency_list', 'adjacency_weights', 'graph_nodes_list', 'graph_state_keep_prob'):
            self.placeholders[k] = k
        dev = self.device

        def var(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev).requires_grad_(True)

        L = self.params['num_timesteps']
        self.weights['edge_weights'] = [var(glorot_init((h_dim, h_dim))) for _ in range(L)]                # gcn:52-53
        if self.params['gcn_use_bias']:
            self.weights['edge_biases'] = [var(np.zeros([h_dim])) for _ in range(L)]                       # gcn:55-57
        # Hidden sizes that are not multiples of 4 run zero-padded at the engine boundary, as in the sparse GGNN plug-in: padded state
        # columns, kernel rows / columns and bias entries are zero, so padded units stay exactly 0 (relu(0) = 0) and add nothing to the
        # real units' sums.  Variables keep the reference's shapes.
        self._padded_hidden = (h_dim + 3) // 4 * 4
        if self.attention_tensor_cores:
            raise Exception("--attention-tensor-cores applies to the sparse GGNN model's propagation attention; the GCN model has none")
        if self.cudnn_gru_tensor_cores:
            raise Exception("--cudnn-gru-tensor-cores applies to the sparse GGNN model's CudnnCompatibleGRUCell; the GCN model has no RNN cell")
        wide = {'wide_hidden': True} if self.gcn_wide_hidden else {}   # the keyword only when the option was given
        self.engine = GCNEngine(self._padded_hidden, L, self.params['gcn_use_bias'], device=self.device.index or 0,
                                precision=self.precision, **wide)
        self._apply_backward_precision(self.engine)
        self._propagation = _propagation_function()
        self._readout = gated_readout_function()

    def graph_model_variables(self):
        """(name, tensor) with the names TensorFlow 1.3 gives the reference's variables: tf.Variable names under the variable scopes
        graph_model (chem_tensorflow.py:141) / gcn_scope (gcn:51)."""
        out = [("graph_model/gcn_scope/gcn_weights_%i:0" % l, w) for l, w in enumerate(self.weights['edge_weights'])]
        out += [("graph_model/gcn_scope/gcn_bias_%i:0" % l, b) for l, b in enumerate(self.weights.get('edge_biases', []))]
        return out

    # ------------------------------------------------------------------ hook 2 (gcn:59-82)
    def compute_final_node_representations(self):
        import torch
        feed = self.feed
        D, DP = self.params['hidden_size'], self._padded_hidden
        h0 = self.initial_node_representation_tensor()
        # a device-data batch was assembled on the device by forward_batch (_adopt_dataset_batch)
        if not feed.get('_graph_adopted'):
            self.engine.set_save_for_backward(torch.is_grad_enabled())   # before set_graph: the source-keyed CSR is built there
        adjacency_weights = None   # a device-built batch's weights: the autograd node's trailing input
        if not feed.get('_graph_adopted') and not self._adopt_prepared_graph(feed):
            lst, w = feed[self.placeholders['adjacency_list']], feed[self.placeholders['adjacency_weights']]
            if isinstance(lst, torch.Tensor) and lst.is_cuda:
                # a list already on the GPU (a device data pipeline, graphs built by torch ops): the batch is built there
                # (set_graph_gcn_device, the host builder's plan and image) and its weights are device data, so a requires_grad tensor
                # gets its gradient and a plain one costs no d w
                dev = torch.device('cuda', self.engine.device)
                self.engine.set_graph_gcn_device(h0.shape[0], lst.to(dev, torch.int64).reshape(-1, 2).contiguous())
                adjacency_weights = (w if isinstance(w, torch.Tensor) else torch.as_tensor(w)).to(dev, torch.float32).contiguous()
            else:
                self.engine.set_graph_gcn(h0.shape[0], lst, w)
        # tf.nn.dropout after the ReLU of every layer but the last (gcn:75-78): done inside the kernels; a fresh mask seed per run, drawn
        # from torch's generator (seeded by params['random_seed'] like tf.set_random_seed, chem_tensorflow.py:85)
        keep = float(feed.get(self.placeholders['graph_state_keep_prob'], 1.0))
        self.engine.set_state_dropout(keep, int(torch.randint(0, 2 ** 62, (1,)).item()) if keep < 1.0 else 0)
        weights = list(self.weights['edge_weights']) + list(self.weights.get('edge_biases', []))
        aw = [adjacency_weights] if adjacency_weights is not None else []
        if DP != D:
            pad = torch.nn.functional.pad
            weights = [pad(w, (0, DP - D) if w.dim() == 1 else (0, DP - D, 0, DP - D)) for w in weights]
            return self._propagation.apply(self.engine, pad(h0, (0, DP - D)).contiguous(), *weights, *aw)[:, :D]
        return self._propagation.apply(self.engine, h0, *weights, *aw)                                     # [V, D]

    # ------------------------------------------------------------------ readout (gcn:84-93 == sparse:220-231)
    gated_regression = SparseGGNNChemModel.gated_regression
    _set_readout_map = SparseGGNNChemModel._set_readout_map

    # ------------------------------------------------------------------ prediction (the sparse model's, sparse:352-376)
    evaluate_one_batch = SparseGGNNChemModel.evaluate_one_batch
    example_evaluation = SparseGGNNChemModel.example_evaluation

    def _prediction_batches(self, raw_graphs, batch_size: int, device_data: bool):
        def host_feed(b):
            feed = dict(b)
            eng = getattr(self, 'engine', None)
            if hasattr(eng, 'prepare_graph_gcn'):   # the host half in this producer thread, as in training
                feed['_prepared_graph'] = self._prepare_from_pool(
                    lambda reuse: eng.prepare_graph_gcn(b['initial_node_representation'].shape[0], b['adjacency_list'], b['adjacency_weights'],
                                                        save_for_backward=False, reuse=reuse), False)
            return feed
        flat = packing.FlatGCNGraphs(packing.process_raw_graphs_gcn(raw_graphs, self.params['task_ids'], labels=False))
        return self._flat_prediction_batches(flat, batch_size, device_data, host_feed)

    # ------------------------------------------------------------------ data (gcn:96-199) via packing.py
    def process_raw_graphs(self, raw_data: Sequence[Any], is_training_data: bool) -> Any:
        processed = packing.process_raw_graphs_gcn(raw_data, self.params['task_ids'])
        if is_training_data:
            np.random.shuffle(processed)                                                         # gcn:106
            for task_id in self.params['task_ids']:
                ratio = self.params['task_sample_ratios'].get(str(task_id))
                if ratio is not None:
                    for ex_id in range(int(len(processed) * ratio), len(processed)):             # gcn:107-112
                        processed[ex_id]['labels'][task_id] = None
        return processed

    def make_minibatch_iterator(self, data: Any, is_training: bool):
        if is_training:
            np.random.shuffle(data)                                                              # gcn:147-148
        keep = self.params['graph_state_dropout_keep_prob'] if is_training else 1.                # gcn:149
        # flattened once per dataset (packing.FlatGCNGraphs); every batch is then a handful of NumPy gathers instead of the per-graph loop
        # of gcn:150-197 -- same arrays, bit for bit, under the same strict node_offset + n < batch_size rule
        flat, order = self._flat_view(data, packing.FlatGCNGraphs)
        if getattr(self, 'device_data', False):   # the same batches, assembled on the device from the uploaded list (forward_batch adopts them)
            for ids in flat.iter_batch_ids(order, self.params['batch_size']):
                yield {'num_graphs': len(ids), 'graph_state_keep_prob': keep, '_graph_sizes': flat.n_nodes[ids],
                       '_dataset_batch': self._dataset_batch(flat, ids, is_training)}
            return
        for b in flat.iter_minibatches(order, self.params['batch_size'], self.params['hidden_size']):
            feed = dict(b, graph_state_keep_prob=keep)
            # this generator runs in ChemModel.run_epoch's ThreadedIterator (chem_tensorflow.py:225): the engine's host half of the batch
            # (index validation, stable CSR by output row, tile plan, one pinned image) is built here, so hook 2 only enqueues the upload
            eng = getattr(self, 'engine', None)
            if getattr(self, 'prepare_graphs_in_producer', True) and hasattr(eng, 'prepare_graph_gcn'):
                feed['_prepared_graph'] = self._prepare_from_pool(
                    lambda reuse: eng.prepare_graph_gcn(b['initial_node_representation'].shape[0], b['adjacency_list'], b['adjacency_weights'],
                                                        save_for_backward=is_training, reuse=reuse), is_training)
            yield feed
