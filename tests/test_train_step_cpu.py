"""CPU: ChemModel.train_step against a float64 restatement of the reference's training op (chem_tensorflow.py:183-191):
tf.clip_by_norm on every variable's gradient, then TensorFlow 1.3's ApplyAdam

    m <- b1 m + (1 - b1) g        v <- b2 v + (1 - b2) g^2        var <- var - lr sqrt(1 - b2^t) / (1 - b1^t) * m / (sqrt(v) + eps)

with tf.train.AdamOptimizer's defaults.  The gradients are the ones loss.backward() leaves in ``p.grad`` (before the clip), so only the
clip and the optimizer are under test; the engine is the oracle-backed stand-in of test_chem_model_cpu.py.  torch's own Adam puts eps
next to sqrt(v / (1 - b2^t)) instead: for gradients below ~1e-4 its steps are visibly larger than TensorFlow's."""
import numpy as np
import pytest

from gated_graph_neural_network_samples_b200 import chem_sparse, synthetic
from tests.test_chem_model_cpu import _args, stand_in  # noqa: F401  (stand_in is a fixture)

B1, B2, EPS = 0.9, 0.999, 1e-8
BAR = 1e-6


def _model(tmp_path, mols):
    np.random.seed(0)
    return chem_sparse.SparseGGNNChemModel(_args(tmp_path, mols, learning_rate=0.001, clamp_gradient_norm=1.0))


def _tf_train_step(var, m, v, g, t, lr, clamp):
    g = g * clamp / max(float(np.sqrt(np.sum(g * g))), clamp)                           # tf.clip_by_norm
    m = B1 * m + (1.0 - B1) * g
    v = B2 * v + (1.0 - B2) * g * g
    lr_t = lr * np.sqrt(1.0 - B2 ** t) / (1.0 - B1 ** t)
    return var - lr_t * m / (np.sqrt(v) + EPS), m, v


def _snapshot(model):
    """float64 copies of every trainable and its Adam slots (zeros before the first update), and the step the next update takes."""
    out, step = {}, 0
    for n, p in model._train_vars:
        st = model.optimizer.state.get(p)
        slot = (lambda k: st[k].detach().double().numpy().copy()) if st else (lambda k: np.zeros(tuple(p.shape)))
        out[n] = (p.detach().double().numpy().copy(), slot("exp_avg"), slot("exp_avg_sq"))
        step = int(st["step"]) if st else 0
    return out, step + 1


def _disagreement(tag, got, ref, before, grad):
    """None when got matches ref to BAR relative to max|ref|; else the worst elements with their gradient and both updates."""
    err = np.abs(got - ref)
    scale = max(float(np.max(np.abs(ref))), 1e-30)
    if float(np.max(err)) <= BAR * scale:
        return None
    worst = np.argsort(err.reshape(-1))[::-1][:4]
    rows = ["%s%s: grad %.3e, update got %.6e, TF %.6e" % (tag, [int(j) for j in np.unravel_index(i, got.shape)], grad.reshape(-1)[i],
                                                           (got - before).reshape(-1)[i], (ref - before).reshape(-1)[i]) for i in worst]
    return "%s max|err|/max|ref| %.2e:\n  %s" % (tag, float(np.max(err)) / scale, "\n  ".join(rows))


def _step_and_check(model, feed):
    """One forward_batch + train_step on ``feed``; every trainable and both its Adam slots against _tf_train_step."""
    before, t = _snapshot(model)
    grads = {}
    hooks = [p.register_post_accumulate_grad_hook(lambda q, n=n: grads.__setitem__(n, q.grad.detach().double().numpy().copy()))
             for n, p in model._train_vars]
    try:
        loss, _ = model.forward_batch(feed)
        model.train_step(loss)
    finally:
        for h in hooks:
            h.remove()
    assert sorted(grads) == sorted(before), "a trainable got no gradient"
    after, t_next = _snapshot(model)
    assert t_next == t + 1
    lr, clamp = model.params["learning_rate"], model.params["clamp_gradient_norm"]
    bad = []
    for n, (var, m, v) in before.items():
        ref = _tf_train_step(var, m, v, grads[n], t, lr, clamp)
        for tag, got, r, prev in zip((n, n[:-2] + "/Adam:0", n[:-2] + "/Adam_1:0"), after[n], ref, before[n]):
            msg = _disagreement(tag, got, r, prev, grads[n])
            if msg:
                bad.append(msg)
    assert not bad, "Adam step %d differs from TensorFlow's ApplyAdam on %d arrays:\n%s" % (t, len(bad), "\n".join(bad))
    return t


def test_three_consecutive_steps_match_tensorflow_adam(tmp_path, stand_in):
    mols = synthetic.make_molecules(64, seed=1)
    model = _model(tmp_path, mols)
    feeds = iter(model.make_minibatch_iterator(model.train_data, True))
    assert [_step_and_check(model, next(feeds)) for _ in range(3)] == [1, 2, 3]


def test_a_step_after_a_checkpoint_restored_at_adam_step_2000(tmp_path, stand_in):
    """The bias corrections of step 2001 are nearly 1 (1 - b1^t) and 0.865 (1 - b2^t): the counter, m and v all come from the pickle."""
    mols = synthetic.make_molecules(64, seed=1)
    model = _model(tmp_path, mols)
    feeds = list(model.make_minibatch_iterator(model.train_data, True))
    _step_and_check(model, feeds[0])
    for st in model.optimizer.state.values():
        st["step"].fill_(2000.0)
    path = str(tmp_path / "adam2000.pickle")
    model.save_progress(path, 2000, 0)
    restored = _model(tmp_path, mols)
    restored.restore_progress(path)
    assert _step_and_check(restored, feeds[1]) == 2001
