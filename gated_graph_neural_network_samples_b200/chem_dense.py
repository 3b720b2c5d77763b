"""``DenseGGNNChemModel`` (chem_tensorflow_dense.py:52-265) on the H100 engine: same hooks, params and feed slots.
The dense model is the engine's dense-adjacency mode: one layer of ``num_timesteps`` steps, A_t . (h W_t + b_t)
computed as (A_t h) W_t + rowsum(A_t) b_t, GRU/tanh, padded rows updated like real ones (dense:100-116)."""
from __future__ import annotations

from collections import defaultdict
from typing import Any, Sequence

import numpy as np

from . import packing
from .chem_model import ChemModel
from .chem_sparse import _propagation_function
from .readout import gated_readout_function
from .engine import PropagationEngine
from .utils import glorot_init
from .workloads import dense_engine_params


def propagate(engine: PropagationEngine, h0, layer: dict, adjacency):
    """The dense GGNN propagation as a differentiable torch function, without a ChemModel: ``engine`` holds a batch of
    ``prepare_graph_dense_device(b, v)`` (adopted with ``set_graph_prepared``), ``h0`` [b*v, D], ``layer`` a dict of fp32 CUDA tensors keyed
    like ``ggnn_layer_weights`` (``engine.WEIGHT_FIELDS``) and ``adjacency`` the fp32 CUDA ``[b, T, v, v]`` matrix, ``A[g, t, i, j]`` the
    weight of the type-t message from node j to node i of graph g (any finite values).  Returns the final node states [b*v, D]; gradients
    reach ``h0``, every layer tensor and every entry of ``adjacency``."""
    lay, flat = {}, []
    for k, v in layer.items():
        lay[k] = len(flat)
        flat.append(v)
    return _propagation_function().apply(engine, [lay], h0, *flat, adjacency)


class DenseGGNNChemModel(ChemModel):
    @classmethod
    def default_params(cls):
        params = dict(super().default_params())
        params.update({'batch_size': 256, 'graph_state_dropout_keep_prob': 1., 'task_sample_ratios': {},   # dense:59-65
                       'use_edge_bias': True, 'edge_weight_dropout_keep_prob': 1})
        return params

    def prepare_specific_graph_model(self) -> None:   # dense:68-91
        import torch
        h_dim, T = self.params['hidden_size'], self.num_edge_types
        for k in ('graph_state_keep_prob', 'edge_weight_dropout_keep_prob', 'initial_node_representation', 'node_mask',
                  'num_vertices', 'adjacency_matrix'):
            self.placeholders[k] = k
        dev = self.device

        def var(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev).requires_grad_(True)

        self.weights['edge_weights'] = var(glorot_init([T, h_dim, h_dim]))                       # dense:84
        if self.params['use_edge_bias']:
            self.weights['edge_biases'] = var(np.zeros([T, 1, h_dim]))                           # dense:86
        self.weights['node_gru'] = {'gate_kernel': var(glorot_init([2 * h_dim, 2 * h_dim])), 'gate_bias': var(np.ones(2 * h_dim)),
                                    'cand_kernel': var(glorot_init([2 * h_dim, h_dim])), 'cand_bias': var(np.zeros(h_dim))}
        # hidden sizes that are not multiples of 4 run zero-padded at the engine boundary (see SparseGGNNChemModel.prepare_specific_graph_model)
        self._padded_hidden = (h_dim + 3) // 4 * 4
        if self.attention_tensor_cores:
            raise Exception("--attention-tensor-cores applies to the sparse GGNN model's propagation attention; the dense model has none")
        if self.cudnn_gru_tensor_cores:
            raise Exception("--cudnn-gru-tensor-cores applies to the sparse GGNN model's CudnnCompatibleGRUCell; the dense model has no cell option")
        if self.gcn_wide_hidden:
            raise Exception("--gcn-wide-hidden applies to the sparse GCN model's hidden sizes; the dense model runs hidden sizes up to 512 "
                            "without it")
        self.engine = PropagationEngine(dense_engine_params(dict(self.params, hidden_size=self._padded_hidden)), T,
                                        device=self.device.index or 0, precision=self.precision)
        self._apply_backward_precision(self.engine)
        self._propagation = _propagation_function()
        self._readout = gated_readout_function()

    def graph_model_variables(self):
        # TF-1.3 names of the dense graph's variables: the two unnamed tf.Variables of dense:84-86 become graph_model/Variable[_1], the
        # GRUCell's variables are created by its first call under graph_model/gru_scope (dense:99).  Restated from knowledge of that release.
        out = [("graph_model/Variable:0", self.weights['edge_weights'])]                         # [T, D, D]
        if 'edge_biases' in self.weights:
            out.append(("graph_model/Variable_1:0", self.weights['edge_biases']))              # [T, 1, D]
        tf_cell = {'gate_kernel': 'gru_cell/gates/kernel', 'gate_bias': 'gru_cell/gates/bias',
                   'cand_kernel': 'gru_cell/candidate/kernel', 'cand_bias': 'gru_cell/candidate/bias'}
        out += [("graph_model/gru_scope/%s:0" % tf_cell[k], v) for k, v in self.weights['node_gru'].items()]
        return out

    def compute_final_node_representations(self):     # dense:93-117
        import torch
        feed = self.feed
        T, D = self.num_edge_types, self.params['hidden_size']
        device_adj = None
        if feed.get('_graph_adopted'):   # a device-data batch, assembled on the device by forward_batch (_adopt_dataset_batch)
            b, v = int(feed[self.placeholders['num_graphs']]), int(feed[self.placeholders['num_vertices']])
        elif isinstance(feed[self.placeholders['adjacency_matrix']], torch.Tensor):
            # a torch tensor (a computed or learned adjacency, [b, e, v, v]): the batch is planned from its shape, the matrix goes to the
            # engine's device as it is (ggnn_set_message_weights) and whatever produced it gets its gradient
            device_adj = feed[self.placeholders['adjacency_matrix']].to(self.device, torch.float32).contiguous()
            b, v = device_adj.shape[0], device_adj.shape[2]
            self.engine.set_save_for_backward(torch.is_grad_enabled())
            self._dense_device_graph = self.engine.prepare_graph_dense_device(b, v, reuse=getattr(self, '_dense_device_graph', None))
            self.engine.set_graph_prepared(self._dense_device_graph)
        else:
            adj = np.asarray(feed[self.placeholders['adjacency_matrix']], dtype=np.float32)      # [b, e, v, v]
            b, v = adj.shape[0], adj.shape[2]
            self.engine.set_save_for_backward(torch.is_grad_enabled())
            if not self._adopt_prepared_graph(feed):     # a graph built by the batch producer thread leaves only the upload
                self.engine.set_graph_dense(adj)
        keep = float(feed.get(self.placeholders['edge_weight_dropout_keep_prob'], 1.0))
        edge_weights = self.weights['edge_weights']
        if keep < 1.0:
            # dense:104 builds a fresh tf.nn.dropout on W[e] per timestep and type.  The engine takes the weights once per sess.run, so the
            # mask is drawn once per batch (every type its own slice of it) and shared by the timesteps -- the sparse model's behaviour
            # (sparse:91).  A deliberate deviation (DESIGN.md 3): the reference feeds this slot with graph_state_dropout_keep_prob
            # (dense:222), so refusing it would make state dropout unusable in dense training.
            edge_weights = torch.nn.functional.dropout(edge_weights, p=1.0 - keep, training=True)
        state_keep = float(feed.get(self.placeholders['graph_state_keep_prob'], 1.0))          # DropoutWrapper, dense:89
        self.engine.set_state_dropout(state_keep, int(torch.randint(0, 2 ** 62, (1,)).item()) if state_keep < 1.0 else 0)
        flat, lay = [edge_weights], {'edge_weights': 0}
        if 'edge_biases' in self.weights:
            lay['edge_biases'] = len(flat); flat.append(self.weights['edge_biases'].view(T, D))
        for k, t in self.weights['node_gru'].items():
            lay[k] = len(flat); flat.append(t)
        h0 = self.initial_node_representation_tensor().reshape(b * v, D)                         # dense:97
        DP = getattr(self, '_padded_hidden', D)
        adj = [] if device_adj is None else [device_adj]   # the trailing message-weight slot of the autograd node
        if DP != D:
            from .chem_sparse import SparseGGNNChemModel
            flat = [SparseGGNNChemModel._pad_hidden(k, flat[i], D, DP) for k, i in lay.items()]
            h0 = torch.nn.functional.pad(h0, (0, DP - D)).contiguous()
            return self._propagation.apply(self.engine, [lay], h0, *flat, *adj)[:, :D].reshape(b, v, D)
        out = self._propagation.apply(self.engine, [lay], h0, *flat, *adj)
        return out.reshape(b, v, D)                                                              # dense:116

    def gated_regression(self, last_h, regression_gate, regression_transform):   # dense:119-129
        import torch
        D = self.params['hidden_size']
        h0 = self.initial_node_representation_tensor().reshape(last_h.shape)   # a device-data batch's h0 is [b*v, D]
        fused = last_h.is_cuda and getattr(self, '_padded_hidden', D) == D   # affine() draws the weight-dropout mask: only when it is used
        ag = regression_gate.affine() if fused and hasattr(regression_gate, 'affine') else None
        at = regression_transform.affine() if fused and hasattr(regression_transform, 'affine') else None
        if ag is not None and at is not None:   # fused kernel (SURVEY 8f-1): masked per-graph sum included
            b, v = last_h.shape[0], last_h.shape[1]
            if not self.feed.get('_graph_adopted'):   # a device-data batch set the readout map and mask with its graph
                self._set_readout_map()
            self.output = self._readout.apply(self.engine, last_h.reshape(b * v, D), h0.reshape(b * v, D), ag[0], ag[1], at[0], at[1])
            return self.output
        gate_input = torch.cat([last_h, h0], dim=2).reshape(-1, 2 * D)
        gated = torch.sigmoid(regression_gate(gate_input)) * regression_transform(last_h.reshape(-1, D))
        gated = gated.reshape(last_h.shape[0], last_h.shape[1])
        mask = self._as_device_tensor(self.feed[self.placeholders['node_mask']])
        self.output = (gated * mask).sum(dim=1)
        return self.output

    def _set_readout_map(self) -> None:
        import torch
        mask = self.feed[self.placeholders['node_mask']]
        if not (torch.is_tensor(mask) and mask.is_cuda):   # a CUDA mask goes as it is: the map is built on the device
            mask = np.asarray(mask, dtype=np.float32)
        self.engine.readout_set_graphs(mask.shape[0], nodes_per_graph=mask.shape[1], node_mask=mask)

    # ------------------------------------------------------------------ prediction (dense:230-265)
    def _prediction_batches(self, raw_graphs, batch_size: int, device_data: bool):
        """The bucketed batches of packing.bucket_batches, packed without targets on the host or assembled from a target-free device dataset."""
        ds = None
        if device_data:
            from .engine import DeviceDataset
            ds = DeviceDataset.for_engine(self.engine, packing.FlatDenseGraphs(raw_graphs, (), self.params['tie_fwd_bkwd']), for_training=False,
                                          stream=0)
        for v, ids in packing.bucket_batches(raw_graphs, batch_size):
            if ds is not None:
                yield {'num_graphs': len(ids), 'num_vertices': v, '_dataset_batch': self._pooled_dataset_batch(ds, ids, False, nodes_per_graph=v)}, ids
                continue
            feed = packing.pack_dense_batch([raw_graphs[i] for i in ids], v, self.params['hidden_size'], self.num_edge_types, (),
                                            self.params['tie_fwd_bkwd'])
            eng = getattr(self, 'engine', None)
            if hasattr(eng, 'prepare_graph_dense'):   # the host half in this producer thread, as in training
                feed['_prepared_graph'] = self._prepare_from_pool(
                    lambda reuse: eng.prepare_graph_dense(feed['adjacency_matrix'], save_for_backward=False, reuse=reuse), False)
            yield feed, ids

    def evaluate_one_batch(self, initial_node_representations, adjacency_matrices, node_masks=None):
        """dense:230-249: one batch of ``b`` graphs -- their node annotations (``b`` lists of rows; the batch has as many rows per graph as
        the first), ``[b, T, v, v]`` adjacency matrices and optionally ``[b, v]`` node masks, by default 1 for each graph's given rows and 0
        beyond, as the reference builds it -- run as in validation.  Returns the reference's fetch ``self.output``: the readout of the LAST
        task of ``task_ids`` only, ``[b]``.  ``predict`` gives every task."""
        import torch
        num_vertices = len(initial_node_representations[0])
        if node_masks is None:
            node_masks = [[1. for _ in r] + [0. for _ in range(num_vertices - len(r))] for r in initial_node_representations]
        b = len(initial_node_representations)
        h0 = np.zeros((b, num_vertices, self.params['hidden_size']), np.float32)   # pad_annotations, dense:166-169
        for i, r in enumerate(initial_node_representations):
            a = np.asarray(r, dtype=np.float32).reshape(len(r), -1)
            h0[i, :a.shape[0], :a.shape[1]] = a
        feed = {'initial_node_representation': h0, 'num_graphs': b, 'num_vertices': num_vertices,
                'adjacency_matrix': np.asarray(adjacency_matrices, dtype=np.float32), 'node_mask': np.asarray(node_masks, dtype=np.float32),
                'graph_state_keep_prob': 1.0, 'out_layer_dropout_keep_prob': 1.0, 'edge_weight_dropout_keep_prob': 1.0}
        with torch.inference_mode():
            return self._last_task_output(self._final_node_representations(feed)).cpu().numpy()

    def example_evaluation(self, valid_file: str = 'molecules_valid.json', n: int = 10):
        """dense:251-265: the targets of the first ``n`` molecules of ``valid_file``, then the predictions of one batch of them in the single
        bucket [29] (rows padded to 29, so the default mask of evaluate_one_batch counts every row, as the reference's does)."""
        import json
        with open(valid_file, 'r') as fh:
            example_molecules = json.load(fh)[:n]
        for mol in example_molecules:
            print(mol['targets'])
        bucketed, bucket_sizes, _ = self.process_raw_graphs(example_molecules, is_training_data=False, bucket_sizes=np.array([29]))
        elements = bucketed[0]
        batch = packing.pack_dense_batch(elements, 29, self.annotation_size, self.num_edge_types, (), self.params['tie_fwd_bkwd'])
        out = self.evaluate_one_batch(list(batch['initial_node_representation']), batch['adjacency_matrix'])
        print(out)
        return out

    def process_raw_graphs(self, raw_data: Sequence[Any], is_training_data: bool, bucket_sizes=None) -> Any:   # dense:132-164
        if bucket_sizes is None:
            bucket_sizes = packing.DEFAULT_BUCKET_SIZES
        bucketed = defaultdict(list)
        for d in raw_data:
            # arrays once, not once per batch: pack_dense_batch's np.asarray calls become no-ops (the dicts themselves are copies)
            d = dict(d, graph=np.asarray(d['graph'], dtype=np.int64).reshape(-1, 3), node_features=np.asarray(d['node_features'], dtype=np.float32))
            bucketed[packing.choose_bucket(d['graph'], bucket_sizes)].append(d)
        if is_training_data:
            for _, bucket in bucketed.items():
                np.random.shuffle(bucket)
                # dense:153-158: beyond the first len(bucket) * ratio examples of the (shuffled) bucket the task's label is dropped
                for task_id in self.params['task_ids']:
                    ratio = self.params.get('task_sample_ratios', {}).get(str(task_id))
                    if ratio is not None:
                        for ex_id in range(int(len(bucket) * ratio), len(bucket)):
                            targets = [list(t) for t in bucket[ex_id]['targets']]
                            targets[task_id][0] = None
                            bucket[ex_id] = dict(bucket[ex_id], targets=targets)
        bucket_at_step = [[idx for _ in range(len(b) // self.params['batch_size'])] for idx, b in bucketed.items()]
        bucket_at_step = [x for y in bucket_at_step for x in y]
        return (bucketed, bucket_sizes, bucket_at_step)

    def make_minibatch_iterator(self, data, is_training: bool):   # dense:194-228
        bucketed, bucket_sizes, bucket_at_step = data
        if is_training:
            np.random.shuffle(bucket_at_step)
            for _, b in bucketed.items():
                np.random.shuffle(b)
        counters = defaultdict(int)
        keep = self.params['graph_state_dropout_keep_prob'] if is_training else 1.
        device_data = getattr(self, 'device_data', False)
        if device_data:
            # --device-data: one dataset of every bucket's graphs, uploaded once; after the same shuffles as above, a batch's graphs are
            # found by identity (their flat ids) and the batch is assembled on the device (forward_batch adopts it)
            keys = list(bucketed)
            flat, order = self._flat_view([g for k in keys for g in bucketed[k]], lambda d: packing.FlatDenseGraphs(
                d, self.params['task_ids'], self.params['tie_fwd_bkwd']), key=bucketed)
            first = dict(zip(keys, np.cumsum([0] + [len(bucketed[k]) for k in keys]).tolist()))
        for bucket in bucket_at_step:
            start = counters[bucket] * self.params['batch_size']
            elements = bucketed[bucket][start:start + self.params['batch_size']]
            if device_data:
                counters[bucket] += 1
                v, ids = int(bucket_sizes[bucket]), order[first[bucket] + start:first[bucket] + start + len(elements)]
                yield {'num_graphs': len(ids), 'num_vertices': v, 'graph_state_keep_prob': keep, 'edge_weight_dropout_keep_prob': keep,
                       '_dataset_batch': self._dataset_batch(flat, ids, is_training, nodes_per_graph=v)}
                continue
            feed = packing.pack_dense_batch(elements, int(bucket_sizes[bucket]), self.params['hidden_size'], self.num_edge_types,
                                            self.params['task_ids'], self.params['tie_fwd_bkwd'])
            feed['graph_state_keep_prob'] = keep
            feed['edge_weight_dropout_keep_prob'] = keep
            counters[bucket] += 1
            # as in the sparse plug-in: this generator runs in run_epoch's ThreadedIterator (chem_tensorflow.py:225), so the engine's host
            # half of the batch (0/1 adjacency -> edge lists -> CSR, tile plan, one pinned image) is built here, next to the packing
            eng = getattr(self, 'engine', None)
            if getattr(self, 'prepare_graphs_in_producer', True) and hasattr(eng, 'prepare_graph_dense'):
                feed['_prepared_graph'] = self._prepare_from_pool(
                    lambda reuse: eng.prepare_graph_dense(feed['adjacency_matrix'], save_for_backward=is_training, reuse=reuse), is_training)
            yield feed
