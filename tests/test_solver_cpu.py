"""CPU-side tests (-m "not gpu") of the solver (3dssd_b200/solver.py, oracle/solver.py, DESIGN.md section 3.11): the two
step-driven schedules, the float32 Adam recipe against float64 and against torch's Adam, the flat parameter buffer, the
layout of the operand arena, and checkpoints by TF variable name."""
import importlib

import numpy as np
import pytest
import torch

from oracle import solver as O

F = np.float32
SOLVER = importlib.import_module("3dssd_b200.solver")


@pytest.fixture(scope="module")
def S():
    return SOLVER


def _model(pkg, arch=None):
    arch = pkg.config.ARCH_3DSSD if arch is None else arch
    d = pkg.params.init_params(arch, 1, seed=5, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=6))
    return d


def test_schedules_of_the_shipped_recipe(S):
    s = S.Solver()
    assert s.learning_rate(0) == F(0.002) and s.learning_rate(64560) == F(0.002)
    assert s.learning_rate(64561) == F(0.002 * 0.1 ** 1) and s.learning_rate(80699) == F(0.002 * 0.1 ** 1)
    assert s.learning_rate(64561) != F(F(0.002) * F(0.1))          # the value is rounded once, from the double product
    assert s.bn_decay(0) == F(0.5) and s.bn_decay(64560) == F(0.5) and s.bn_decay(64561) == F(0.75)
    assert isinstance(s.learning_rate(3), np.float32) and isinstance(s.bn_decay(3), np.float32)
    for step in (0, 1, 64559, 64560, 64561, 10 ** 7):
        assert s.learning_rate(step) == O.learning_rate(step) and s.bn_decay(step) == O.bn_decay(step)


def test_schedules_with_several_boundaries_and_none(S):
    s = S.Solver(steps=(2, 5, 9), gamma=0.5)
    want = [F(0.002), F(0.002 * 0.5), F(0.002 * 0.5 ** 2), F(0.002 * 0.5 ** 3)]
    assert [s.learning_rate(t) for t in (0, 2, 3, 5, 6, 9, 10)] == [want[i] for i in (0, 0, 1, 1, 2, 2, 3)]
    assert s.lr_values() == [float(x) for x in want]
    assert [s.bn_decay(t) for t in (2, 3, 6, 10)] == [F(0.5), F(0.75), F(0.875), F(1.0) - F(0.5 * 0.5 ** 3)]
    for t in range(12):
        assert s.learning_rate(t) == O.learning_rate(t, steps=(2, 5, 9), gamma=0.5)
        assert s.bn_decay(t) == O.bn_decay(t, steps=(2, 5, 9))
    c = S.Solver(steps=())
    assert c.learning_rate(0) == c.learning_rate(10 ** 6) == F(0.002) and c.bn_decay(10 ** 6) == F(0.5)
    with pytest.raises(ValueError):
        S.Solver(steps=(5, 5))
    with pytest.raises(ValueError):
        S.Solver(steps=tuple(range(1, 10)))


def test_bn_decay_clip_engages(S):
    s = S.Solver(steps=tuple(range(10, 90, 10)))                     # 1 - 0.5 * 0.5^6 = 0.9922 > 0.99
    assert s.bn_decay(60) == F(1.0) - F(0.5 * 0.5 ** 5) < F(0.99)
    assert s.bn_decay(61) == F(0.99) and s.bn_decay(1000) == F(0.99)


def test_the_misspelt_floor_of_the_reference_is_not_applied(S):
    s = S.Solver(steps=(1, 2, 3), gamma=0.01)
    assert s.learning_rate(4) == F(0.002 * 0.01 ** 3) < F(1e-5)


def _run_oracle(p, grads, boundaries, values):
    st = O.new_state()
    m, v = np.zeros_like(p), np.zeros_like(p)
    for g in grads:
        p, m, v, st = O.adam_step(p, g, m, v, st, boundaries, values)
    return p, m, v, st


def test_oracle_adam_agrees_with_float64():
    rng = np.random.default_rng(0)
    p0 = rng.standard_normal(4096).astype(F)
    grads = [(rng.standard_normal(4096) * 0.1).astype(F) for _ in range(50)]
    p, m, v, st = _run_oracle(p0, grads, (20,), (0.002, 0.0002))
    q, qm, qv = p0.astype(np.float64), np.zeros(4096), np.zeros(4096)
    for t, g in enumerate(grads):
        q, qm, qv = O.adam_step_f64(q, g, qm, qv, t + 1, float(F(0.002)) if t <= 20 else float(F(0.0002)))
    assert st["global_step"] == 50 and st["lr_used"] == F(0.0002)
    assert abs(float(st["beta1_power"]) - 0.9 ** 51) < 1e-6 * 0.9 ** 51 * 51    # the float32 power lags the exact one slightly
    ulp = np.spacing(np.abs(q).astype(F)).astype(np.float64)
    assert (np.abs(p - q) <= 40 * ulp + 2e-7).all()                  # 50 steps of ~lr each: a few ulp per step
    np.testing.assert_allclose(m, qm, rtol=2e-5, atol=5e-8)              # a few ulp of the largest |m| ~ 0.1
    np.testing.assert_allclose(v, qv, rtol=2e-5, atol=1e-9)


def test_torch_adam_is_close_on_ordinary_gradients_but_not_the_same_rule():
    """torch.optim.Adam divides by (sqrt(v) / sqrt(1 - beta2^t) + eps): epsilon INSIDE the bias correction.  TF's
    ApplyAdam folds the correction into alpha and adds epsilon to the raw sqrt(v) ("epsilon hat").  With gradients far
    above epsilon the two agree to about 1e-4 relative; with sqrt(v) near epsilon the steps differ severalfold."""
    def torch_adam(p0, grads, lr):
        t = torch.tensor(p0.copy(), requires_grad=True)
        opt = torch.optim.Adam([t], lr=lr)
        for g in grads:
            t.grad = torch.from_numpy(g.copy())
            opt.step()
        return t.detach().numpy()

    rng = np.random.default_rng(1)
    p0 = rng.standard_normal(512).astype(F)
    grads = [(rng.standard_normal(512) * 0.1).astype(F) for _ in range(10)]
    p = _run_oracle(p0, grads, (), (0.002,))[0]
    np.testing.assert_allclose(p - p0, torch_adam(p0, grads, 0.002) - p0, rtol=1e-3, atol=1e-6)   # atol: 10 roundings of p ~ 1
    tiny = [np.full(512, 1e-9, F)]                                   # sqrt(v) = 1e-9 * sqrt(0.001) = 3e-11 << epsilon
    ours = _run_oracle(p0, tiny, (), (0.002,))[0] - p0
    theirs = torch_adam(p0, tiny, 0.002) - p0
    want = -0.002 * np.sqrt(0.001) / 0.1 * (1e-10 / (1e-9 * np.sqrt(0.001) + 1e-8))     # TF's rule in double
    np.testing.assert_allclose(ours, want, rtol=0.05, atol=2e-7)     # atol: the float32 grid of p near 1
    assert abs(np.median(theirs)) > 3 * abs(np.median(ours))


def test_flat_params_keeps_leaves_values_and_grad_offsets(pkg):
    arch = [spec for spec in pkg.config.ARCH_3DSSD][:1]
    d = pkg.params.init_params(arch, 1, seed=2, random_bias=True)
    tp = pkg.params.TrainableParams(d, "cpu")
    before = {k: t.detach().clone() for k, t in tp.named_parameters()}
    ids = {k: id(t) for k, t in tp.named_parameters()}
    flat = tp.flat_params()
    assert tp.flat_params() is flat and flat.dtype == torch.float32 and flat.numel() == sum(t.numel() for t in before.values())
    tp.flat_grads()
    assert tp.param_offsets == tp.grad_offsets and list(tp.param_offsets) == [k for k, _ in tp.named_parameters()]
    for k, t in tp.named_parameters():
        assert id(t) == ids[k] and t.is_leaf and t.requires_grad
        assert torch.equal(t.detach(), before[k])
        o = tp.param_offsets[k]
        assert t.data_ptr() == flat.data_ptr() + 4 * o
        assert t.grad.data_ptr() == tp.grad_flat.data_ptr() + 4 * o
    k = "layer1/conv0_0/weights"
    flat[tp.param_offsets[k]] = 42.0
    assert tp.tensors[k][0, 0].item() == 42.0
    (tp.tensors[k] * 2).sum().backward()                              # still a leaf autograd accumulates into
    assert tp.grad_flat[tp.param_offsets[k]].item() == 2.0
    assert tp.operand_cache is None


def test_operand_arena_layout_of_the_shipped_model(pkg):
    P = pkg.params
    d = _model(pkg)
    weights, off = [], 0
    for k, v in d.items():                                            # named_parameters order = dict order of trainables
        if k.endswith(("/bn/moving_mean", "/bn/moving_variance")):
            continue
        if k.endswith("/weights"):
            weights.append((off,) + v.shape)
        off += v.size
    assert off == 2513858
    table, elems, tiles = P.operand_layout(weights)
    assert table.shape == (len(weights), 8) and table.dtype == np.int64 and len(weights) > 40
    assert {4, 67, 131, 259} <= {w[1] for w in weights}               # the paddings that are not multiples of 16
    spans = []
    for row, (poff, cin, cout) in zip(table, weights):
        assert tuple(row[:3]) == (poff, cin, cout)
        fwd, bwd = cout * P.round16(cin), cin * P.round16(cout)
        for o, size in ((row[3], fwd), (row[4], fwd), (row[5], bwd), (row[6], bwd)):
            assert (2 * o) % 16 == 0                                  # bf16 elements -> bytes
            spans.append((int(o), int(o) + size))
    spans.sort()
    assert spans[0][0] == 0 and spans[-1][1] == elems
    assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))        # back to back: no overlap, no hole
    starts = table[:, 7]
    per = [-(-P.round16(ci) // 32) * -(-P.round16(co) // 32) for _, ci, co in weights]
    assert starts[0] == 0 and (np.diff(starts) == per[:-1]).all() and tiles == starts[-1] + per[-1]


def test_state_block_round_trips(S):
    w = S.pack_state(64561, F(0.9) * F(0.9), F(0.999), F(0.002))
    assert w.dtype == np.int32 and w.shape == (8,) and (w[5:] == 0).all()
    assert S.unpack_state(w) == (64561, F(0.9) * F(0.9), F(0.999), F(0.002))
    assert S.unpack_state(S.pack_state(2 ** 40 + 3, 0.5, 0.25))[0] == 2 ** 40 + 3


def test_checkpoint_variables_round_trip(pkg, S, tmp_path):
    """The serialisation functions on CPU data: what save() writes goes through kitti_io.params_from_tf_variables
    unchanged, the optimizer's part comes back exactly, and a file without a slot is refused."""
    arch = [spec for spec in pkg.config.ARCH_3DSSD][:1]
    d = pkg.params.init_params(arch, 1, seed=4, random_bias=True)
    tp = pkg.params.TrainableParams(d, "cpu")
    tp.flat_params()
    named = [(k, tuple(t.shape)) for k, t in tp.named_parameters()]
    n = tp.param_flat.numel()
    rng = np.random.default_rng(7)
    adam = {"m": rng.standard_normal(n).astype(F), "v": rng.uniform(0, 1, n).astype(F), "global_step": 2421,
            "beta1_power": F(0.123), "beta2_power": F(0.987), "lr_used": F(0.002)}
    variables = S._variables(named, tp.to_params(), tp.param_offsets, adam)
    assert variables["layer1/conv0_0/weights/Adam"].shape == (4, 16) and "layer1/conv0_0/bn/moving_mean/Adam" not in variables
    assert set(variables) == set(d) | {k + s for k, _ in named for s in ("/Adam", "/Adam_1")} | set(S.SCALARS)
    path = tmp_path / "model-00002421.npz"
    np.savez(str(path), **variables)
    with np.load(str(path)) as z:
        got = {k: z[k] for k in z.files}
    params = pkg.kitti_io.params_from_tf_variables(got)
    assert set(params) == set(d)
    for k in d:
        np.testing.assert_array_equal(params[k], d[k])
    back = S._from_variables(named, tp.param_offsets, n, got)
    assert back["global_step"] == 2421 and back["beta1_power"] == F(0.123) and back["beta2_power"] == F(0.987)
    np.testing.assert_array_equal(back["m"], adam["m"]); np.testing.assert_array_equal(back["v"], adam["v"])
    del got["layer1/conv0_0/biases/Adam_1"]
    with pytest.raises(ValueError, match="Adam_1"):
        S._from_variables(named, tp.param_offsets, n, got)


class _StubTrainer(SOLVER.Trainer):
    """Trainer's checkpoint methods over CPU tensors: no kernel runs (the operand cache is off, the Adam state is a dict)."""

    def __init__(self, S, tp):
        self.tp, self.global_step, self.solver = tp, 0, S.Solver()
        tp.flat_params()
        n = tp.param_flat.numel()
        stub = type("A", (), {})()
        stub.param, stub.sd = tp.param_flat, {"m": np.zeros(n, F), "v": np.zeros(n, F), "global_step": 0,
                                              "beta1_power": F(0.9), "beta2_power": F(0.999)}
        stub.state_dict = lambda: stub.sd
        stub.load_state_dict = lambda sd: setattr(stub, "sd", sd)
        self.adam = stub


def test_load_restores_everything_and_warm_start_only_the_model(pkg, S, tmp_path):
    arch = [spec for spec in pkg.config.ARCH_3DSSD][:1]
    a = _StubTrainer(S, pkg.params.TrainableParams(pkg.params.init_params(arch, 1, seed=4, random_bias=True), "cpu"))
    n = a.tp.param_flat.numel()
    rng = np.random.default_rng(3)
    a.adam.sd = {"m": rng.standard_normal(n).astype(F), "v": rng.uniform(0, 1, n).astype(F), "global_step": 807,
                 "beta1_power": F(0.25), "beta2_power": F(0.5)}
    path = str(tmp_path / "a.npz")
    a.save(path)

    b = _StubTrainer(S, pkg.params.TrainableParams(pkg.params.init_params(arch, 1, seed=9), "cpu"))
    flat = b.tp.param_flat
    b.load(path)
    assert b.global_step == 807 and b.adam.sd["global_step"] == 807
    assert b.adam.sd["beta1_power"] == F(0.25) and b.adam.sd["beta2_power"] == F(0.5)
    np.testing.assert_array_equal(b.adam.sd["m"], a.adam.sd["m"]); np.testing.assert_array_equal(b.adam.sd["v"], a.adam.sd["v"])
    assert b.tp.param_flat is flat and torch.equal(flat, a.tp.param_flat)        # written in place: the views stay
    for k, t in a.tp.tensors.items():
        assert torch.equal(b.tp.tensors[k], t), k

    c = _StubTrainer(S, pkg.params.TrainableParams(pkg.params.init_params(arch, 1, seed=9), "cpu"))
    with np.load(path) as z:
        extra = {k: z[k] for k in z.files}
    extra["some/other/model/weights"] = np.zeros((3, 3), F)
    del extra["layer1/conv0_0/biases"]
    keep = c.tp.tensors["layer1/conv0_0/biases"].detach().clone()
    path2 = str(tmp_path / "pretrained.npz")
    np.savez(path2, **extra)
    copied = c.warm_start(path2)
    assert c.global_step == 0 and c.adam.sd["global_step"] == 0 and not c.adam.sd["m"].any()
    assert "layer1/conv0_0/biases" not in copied and len(copied) == len(c.tp.tensors) - 1
    assert torch.equal(c.tp.tensors["layer1/conv0_0/biases"], keep)
    assert torch.equal(c.tp.tensors["layer1/conv0_0/weights"], a.tp.tensors["layer1/conv0_0/weights"])
    assert torch.equal(c.tp.tensors["layer1/conv0_0/bn/moving_mean"], a.tp.tensors["layer1/conv0_0/bn/moving_mean"])
    with pytest.raises(ValueError, match="lacks"):
        c.load(path2)
