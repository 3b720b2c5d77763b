"""Float64 restatement of the GGNN propagation over a dense ``[b, T, v, v]`` adjacency held as a torch tensor (ggnn_prepare_graph_dense_device,
DESIGN §2.14):

    incoming[g*v+i] = sum_t sum_j A[g,t,i,j] (h[g*v+j] W_t + b_t)        (dense:103-113; no averaging)

for every layer of the engine's params (residual inputs, GRU / RNN / CudnnCompatibleGRUCell, state dropout), so that torch autograd gives
the float64 reference of every gradient, ``A``'s included.  With one GRU layer it is ``oracle.ggnn_oracle.dense_propagation_torch``; the
cells, residual selection and dropout mask are the oracle's.  ``adjacency_grad_statement`` restates dA from the recorded steps:

    dA[g,t,i,j] = sum over the timesteps of  <P_t[g*v+i], h[g*v+j]> + <dx'[g*v+i], b_t>,   P_t = dx' W_t^T
"""
import numpy as np

from oracle import ggnn_oracle as O


def propagation_torch(h0, adjacency, weights, params, dtype=None, state_dropout=None, mask_width=None, record=None):
    """``h0`` [b*v, D], ``adjacency`` [b, T, v, v], ``weights`` a list of per-layer dicts in the oracle's format (``rnn_kernel`` /
    ``rnn_bias`` for RNN, ``edge_biases`` [T, D] or [T, 1, D]).  Returns the final states [b*v, D].  ``record`` (a list): every timestep
    appends (h, incoming, W, B) with ``incoming.retain_grad()``, for ``adjacency_grad_statement``."""
    import torch
    assert not params.get("use_edge_msg_avg_aggregation", False) and not params.get("use_propagation_attention", False)
    dtype = dtype or torch.float64
    t = lambda a: a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    h0 = t(h0).to(dtype)
    A = t(adjacency).to(dtype)
    b, T, v, _ = A.shape
    V, D = h0.shape
    act = torch.tanh if params.get("graph_rnn_activation", "tanh").lower() == "tanh" else torch.relu
    cell_type = params.get("graph_rnn_cell", "GRU").lower()
    states = [h0]
    gs = 0
    for layer_idx, num_timesteps in enumerate(params["layer_timesteps"]):
        w = {k: t(x).to(dtype) for k, x in weights[layer_idx].items()}
        B = w["edge_biases"].reshape(T, D) if params.get("use_edge_bias", False) else None
        residual_states = [states[i] for i in O.residual_inputs_of_layer(params, layer_idx)]
        states.append(states[-1])
        for _ in range(num_timesteps):
            h = states[-1]
            incoming = torch.zeros(b, v, D, dtype=dtype)
            for e in range(T):
                m = (h @ w["edge_weights"][e]).reshape(b, v, D)
                if B is not None:
                    m = m + B[e]
                incoming = incoming + torch.matmul(A[:, e], m)
            incoming = incoming.reshape(V, D)
            if record is not None:
                incoming.retain_grad()
                record.append((h, incoming, w["edge_weights"], B))
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


def adjacency_grad_statement(record, b, v):
    """dA [b, T, v, v] from the steps ``propagation_torch`` recorded, after a backward: per step, P_t = dx' W_t^T and
    dA[g,t,i,j] += <P_t[g*v+i], h[g*v+j]> + <dx'[g*v+i], b_t>  (dx' = the recorded incoming's gradient)."""
    import torch
    out = None
    for h, incoming, W, B in record:
        dx = incoming.grad.detach()
        hd = h.detach()
        T, D = W.shape[0], W.shape[-1]
        P = torch.einsum("vk,tmk->tvm", dx, W.detach())                       # P_t[row] = dx'[row] . W_t^T
        term = torch.einsum("tgim,gjm->gtij", P.reshape(T, b, v, D), hd.reshape(b, v, D))
        if B is not None:
            term = term + torch.einsum("gim,tm->gti", dx.reshape(b, v, D), B.detach())[..., None]
        out = term if out is None else out + term
    return out
