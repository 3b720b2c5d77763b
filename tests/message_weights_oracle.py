"""Float64 restatements of the sparse GGNN model with message weights (ggnn_prepare_graph_sparse_weighted / ggnn_set_message_weights):

    incoming[v] = ( sum_t (sum_{m into v, type t} w_m h[s_m]) W_t  +  sum_t indeg[v,t] b_t ) / denom[v]

Message m of type t is at position sum_{t' < t} E_t' + i, the order of ``oracle.ggnn_oracle.message_arrays``.  The weight scales the state
term only; the in-degree table is used as fed.  With ``message_weights=None`` both functions are the oracle's own sparse restatements, and
the cells, residual selection, bias, mean and state dropout are the oracle's (``oracle/ggnn_oracle.py``).  Attention is not restated: the
engine refuses it on a message-weighted batch.
"""
import numpy as np

from oracle import ggnn_oracle as O


def propagation_loops(h0, adjacency_lists, num_incoming_edges_per_type, weights, params, message_weights=None, dtype=np.float64):
    """``O.sparse_propagation_loops`` with message m's state term scaled by ``message_weights[m]``, message by message in message order."""
    if message_weights is None:
        return O.sparse_propagation_loops(h0, adjacency_lists, num_incoming_edges_per_type, weights, params, dtype=dtype)
    assert not params.get("use_propagation_attention", False)
    h0 = np.asarray(h0, dtype=dtype)
    indeg = np.asarray(num_incoming_edges_per_type, dtype=dtype)
    mw = np.asarray(message_weights, dtype=dtype)
    weights = O._cast_weights(weights, dtype)
    V, D = h0.shape
    cell = O._cell_fn(params)
    states = [h0]
    for layer_idx, num_timesteps in enumerate(params["layer_timesteps"]):
        w = weights[layer_idx]
        residual_states = [states[i] for i in O.residual_inputs_of_layer(params, layer_idx)]
        states.append(states[-1])
        for _ in range(num_timesteps):
            h = states[-1]
            incoming = np.zeros((V, D), dtype=dtype)
            m = 0
            for e, adj in enumerate(adjacency_lists):
                for src, tgt in np.asarray(adj).reshape(-1, 2):
                    incoming[tgt] += mw[m] * (h[src] @ w["edge_weights"][e])
                    m += 1
            if params.get("use_edge_bias", False):
                incoming = incoming + indeg @ w["edge_biases"].reshape(-1, D)
            if params.get("use_edge_msg_avg_aggregation", False):
                incoming = incoming / (indeg.sum(axis=-1, keepdims=True) + dtype(O.SMALL_NUMBER))
            states[-1] = cell(np.concatenate(residual_states + [incoming], axis=-1), h, w)
    return states[-1]


def propagation_torch(h0, adjacency_lists, num_incoming_edges_per_type, weights, params, message_weights=None, dtype=None,
                      state_dropout=None, mask_width=None):
    """``O.sparse_propagation_torch`` with the messages scaled by ``message_weights`` before the segment sum: torch tensors with
    ``requires_grad`` (``h0``, the weights, ``message_weights``) give the float64 autograd reference of every gradient."""
    import torch
    if message_weights is None:
        return O.sparse_propagation_torch(h0, adjacency_lists, num_incoming_edges_per_type, weights, params, dtype=dtype,
                                          state_dropout=state_dropout, mask_width=mask_width)
    assert not params.get("use_propagation_attention", False)
    dtype = dtype or torch.float64
    t = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    h0 = t(h0).to(dtype)
    indeg = t(num_incoming_edges_per_type).to(dtype)
    mw = t(message_weights).to(dtype)
    adjs = [torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.int64).reshape(-1, 2))) for a in adjacency_lists]
    V, D = h0.shape
    act = torch.tanh if params.get("graph_rnn_activation", "tanh").lower() == "tanh" else torch.relu
    cell_type = params.get("graph_rnn_cell", "GRU").lower()
    targets = torch.cat([a[:, 1] for a in adjs])
    states = [h0]
    gs = 0
    for layer_idx, num_timesteps in enumerate(params["layer_timesteps"]):
        w = {k: t(v).to(dtype) for k, v in weights[layer_idx].items()}
        residual_states = [states[i] for i in O.residual_inputs_of_layer(params, layer_idx)]
        states.append(states[-1])
        for _ in range(num_timesteps):
            h = states[-1]
            messages = torch.cat([torch.index_select(h, 0, a[:, 0]) @ w["edge_weights"][e] for e, a in enumerate(adjs)], dim=0)
            incoming = torch.zeros(V, D, dtype=dtype).index_add(0, targets, messages * mw.unsqueeze(-1))
            if params.get("use_edge_bias", False):
                incoming = incoming + indeg @ w["edge_biases"].reshape(-1, D)
            if params.get("use_edge_msg_avg_aggregation", False):
                incoming = incoming / (indeg.sum(dim=-1, keepdim=True) + O.SMALL_NUMBER)
            x = torch.cat(residual_states + [incoming], dim=-1)
            if cell_type == "rnn":
                new = act(torch.cat([x, h], -1) @ w["rnn_kernel"] + w["rnn_bias"])
            else:
                ru = torch.sigmoid(torch.cat([x, h], -1) @ w["gate_kernel"] + w["gate_bias"])
                r, u = ru[:, :D], ru[:, D:]
                if cell_type == "gru":
                    c = act(torch.cat([x, r * h], -1) @ w["cand_kernel"] + w["cand_bias"])
                else:   # CudnnCompatibleGRUCell
                    din = x.shape[-1]
                    c = act(x @ w["cand_kernel"][:din] + w["cand_bias"] + r * (h @ w["cand_kernel"][din:] + w["cand_hidden_bias"]))
                new = u * h + (1 - u) * c
            states[-1] = O._apply_state_dropout(new, state_dropout, gs, mask_width)
            gs += 1
    return states[-1]
