"""Autograd node around the fused gated-regression readout of the C ABI (``ggnn_readout_forward/backward``) --
``gated_regression`` of chem_tensorflow_sparse.py:220-231 / chem_tensorflow_dense.py:119-129 for readout MLPs without hidden
layers (what chem_tensorflow.py:153-157 builds)."""
from __future__ import annotations


def gated_readout_function():
    import torch

    class GatedReadout(torch.autograd.Function):
        @staticmethod
        def forward(ctx, engine, h_last, h0, w_gate, b_gate, w_trans, b_trans):
            args = [t.detach().contiguous() for t in (h_last, h0, w_gate, b_gate, w_trans, b_trans)]
            engine.set_deterministic(torch.are_deterministic_algorithms_enabled())
            out = engine.readout_forward(*args)
            ctx.engine, ctx.args = engine, args
            ctx.shapes = (w_gate.shape, b_gate.shape, w_trans.shape, b_trans.shape)
            return out

        @staticmethod
        def backward(ctx, d_out):
            ctx.engine.set_deterministic(torch.are_deterministic_algorithms_enabled())
            d_h, d_wg, d_bg, d_wt, d_bt = ctx.engine.readout_backward(*ctx.args, d_out.contiguous())
            s = ctx.shapes
            return None, d_h, None, d_wg.view(s[0]), d_bg.view(s[1]), d_wt.view(s[2]), d_bt.view(s[3])

    return GatedReadout
