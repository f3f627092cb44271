"""CPU checks of fine-tuning and the Momentum solver (DESIGN.md section 3.19): the TRAIN_PARAM_PREFIX filter on the 3DSSD
variable names, the frozen set of TrainableParams, a float32 restatement of TF's ApplyMomentum across a learning-rate
boundary, the C prototype and argument packing of ssd3d_momentum_step, and checkpoints whose optimizer slots cover the
trained variables only."""
import ctypes
import importlib
import os
import re

import numpy as np
import pytest
import torch

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = importlib.import_module("3dssd_b200.solver")
TOP = ["layer4", "conv1d_0", "pred_"]        # the candidate-generation layer and the head


def momentum_step(p, g, accum, state, boundaries, values, momentum):
    """TF's ApplyMomentum (use_nesterov=False) in float32, each operation rounded once: accum = accum * momentum + g;
    p -= accum * lr, lr = values[number of boundaries < global_step] of the state before the step.  Returns new arrays
    and the new state {global_step, lr_used}."""
    lr = F(values[sum(1 for b in boundaries if state["global_step"] > b)])
    with np.errstate(invalid="ignore", over="ignore"):
        a = (accum.astype(F) * F(momentum)).astype(F) + g.astype(F)
        q = p.astype(F) - (a * lr).astype(F)
    return q.astype(F), a.astype(F), {"global_step": state["global_step"] + 1, "lr_used": lr}


def model(pkg, seed=5):
    arch = pkg.config.ARCH_3DSSD
    d = pkg.params.init_params(arch, 1, seed=seed, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=seed + 1))
    return d


def _trainables(d):
    return [k for k in d if not k.endswith(("/bn/moving_mean", "/bn/moving_variance"))]


def test_prefix_filter_on_the_3dssd_variables(pkg):
    P = pkg.params
    names = _trainables(model(pkg))
    assert P.trained_names(names, []) == names == P.trained_names(names, None)
    top = P.trained_names(names, TOP)
    assert top == [k for k in names if k.split("/")[0] in ("layer4", "conv1d_0", "pred_cls_base", "pred_cls", "pred_reg_base",
                                                           "pred_reg")]
    assert {k.split("/")[0] for k in top} == {"layer4", "conv1d_0", "pred_cls_base", "pred_cls", "pred_reg_base", "pred_reg"}
    assert not any(k.startswith(("layer1", "layer2", "layer3", "vote")) for k in top)
    l1 = P.trained_names(names, ["layer1"])
    assert l1 and all(k.startswith("layer1/") for k in l1) and len(l1) == sum(k.startswith("layer1/") for k in names)
    with pytest.raises(ValueError, match="layer9"):
        P.trained_names(names, ["layer1", "layer9"])
    assert P.trained_names(names, ["pred_cls/"]) == ["pred_cls/weights", "pred_cls/biases"]   # re.match, not a scope name
    assert P.trained_names(names, [r"layer[12]/conv0_0/weights"]) == ["layer1/conv0_0/weights", "layer2/conv0_0/weights"]


def test_trainable_params_freeze_the_rest(pkg):
    d = model(pkg)
    tp = pkg.params.TrainableParams(d, "cpu", trainable=TOP)
    want = pkg.params.trained_names(_trainables(d), TOP)
    assert [k for k, _ in tp.named_parameters()] == want
    assert set(tp.frozen_names()) == set(_trainables(d)) - set(want)
    for k, t in tp.tensors.items():
        assert t.requires_grad == (k in want), k
    flat = tp.flat_params()
    tp.flat_grads()
    assert flat.numel() == sum(d[k].size for k in want) == tp.grad_flat.numel()
    assert list(tp.param_offsets) == want
    assert all(tp.tensors[k].grad is None for k in tp.frozen_names())
    assert tp.weight_scopes() == [k[:-8] for k in want if k.endswith("/weights")]
    full = pkg.params.TrainableParams(d, "cpu")
    assert [k for k, _ in full.named_parameters()] == _trainables(d) and not full.frozen_names()


def test_momentum_recipe_across_a_boundary():
    """The float32 recipe against float64 over 30 steps whose learning rate drops after step 10, and the state it keeps."""
    rng = np.random.default_rng(0)
    n = 4096
    p0 = rng.standard_normal(n).astype(F)
    grads = [(rng.standard_normal(n) * 0.1).astype(F) for _ in range(30)]
    boundaries, values = (10,), (float(F(0.002)), float(F(0.0002)))
    p, a, st = p0, np.zeros(n, F), {"global_step": 0, "lr_used": F(0)}
    q, qa = p0.astype(np.float64), np.zeros(n)
    lrs = []
    for t, g in enumerate(grads):
        p, a, st = momentum_step(p, g, a, st, boundaries, values, 0.9)
        lrs.append(st["lr_used"])
        lr = values[0] if t <= 10 else values[1]
        qa = qa * float(F(0.9)) + g
        q = q - qa * lr
    assert st["global_step"] == 30 and lrs[10] == F(0.002) and lrs[11] == F(0.0002)
    assert np.abs(p - q).max() < 1e-5 and np.abs(a - qa).max() < 1e-5
    p1, a1, _ = momentum_step(p0, grads[0], np.zeros(n, F), {"global_step": 0}, (), (0.002,), 0.9)
    np.testing.assert_array_equal(a1, grads[0])                     # the slot starts at zero: the first step is plain SGD
    np.testing.assert_array_equal(p1, p0 - (grads[0] * F(0.002)).astype(F))
    bad = np.array([np.inf, np.nan, 1.0], F)
    p2, a2, _ = momentum_step(np.zeros(3, F), bad, np.zeros(3, F), {"global_step": 0}, (), (0.002,), 0.9)
    assert np.isinf(a2[0]) and np.isnan(a2[1]) and np.isnan(p2[1]) and np.isfinite(p2[2])


_CTYPES = {"float *": ctypes.c_void_p, "const float *": ctypes.c_void_p, "void *": ctypes.c_void_p, "long": ctypes.c_long,
           "float": ctypes.c_float, "int": ctypes.c_int, "const long long *": ctypes.c_void_p,
           "ssd3d_stream_t": ctypes.c_void_p}


def test_momentum_step_prototype_matches_the_header():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ssd3d.h")).read(), flags=re.S)
    m = re.search(r"int\s+ssd3d_momentum_step\s*\(([^)]*)\)", hdr)
    assert m
    args = [re.sub(r"\s+", " ", a).strip() for a in m.group(1).split(",")]
    types = [re.match(r"(.*?)\w+$", a).group(1).strip() for a in args]          # drop each parameter's name
    L = importlib.import_module("3dssd_b200._lib")
    assert L._SIGNATURES["ssd3d_momentum_step"] == [_CTYPES[t] for t in types], types
    assert "ssd3d_momentum_step" in L.EXPORTS


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a))
            return 0
        return fn


def test_momentum_step_packs_its_arguments(pkg, monkeypatch):
    """tf_ops.momentum_step through a recording library with is_cuda forced on: one call, the buffers' addresses, n, the
    momentum and the schedule as host arrays; malformed operands are refused before anything reaches the library."""
    T = pkg.tf_ops
    rec = _Recorder()
    monkeypatch.setattr(T, "lib", lambda: rec)
    monkeypatch.setattr(T, "_stream", lambda: None)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    p, g, a = torch.zeros(12), torch.zeros(12), torch.zeros(12)
    st = torch.zeros(8, dtype=torch.int32)
    T.momentum_step(p, g, a, st, (3, 7), (0.5, 0.25, 0.125), momentum=0.75)
    assert [c[0] for c in rec.calls] == ["ssd3d_momentum_step"]
    args = rec.calls[0][1]
    assert [args[i].value for i in (0, 1, 2, 4)] == [t.data_ptr() for t in (p, g, a, st)]
    assert args[3] == 12 and args[5] == 0.75 and args[6] == 2
    assert list((ctypes.c_longlong * 2).from_address(args[7].value)) == [3, 7]
    assert list((ctypes.c_float * 3).from_address(args[8].value)) == [0.5, 0.25, 0.125]
    for bad in (lambda: T.momentum_step(p, g, torch.zeros(11), st, (), (0.1,)),
                lambda: T.momentum_step(p, g, a, st, (2, 1), (0.1, 0.1, 0.1)),
                lambda: T.momentum_step(p, g, a, st, (), (0.1, 0.2)),
                lambda: T.momentum_step(p, g, a, st, (), (0.1,), momentum=1.5),
                lambda: T.momentum_step(torch.zeros(13)[1:], g, a, st, (), (0.1,))):
        with pytest.raises(ValueError):
            bad()
    assert len(rec.calls) == 1


def test_solver_types():
    assert S.Solver().type == "adam" and S.Solver(type="momentum").momentum == 0.9
    with pytest.raises(ValueError):
        S.Solver(type="sgd")
    with pytest.raises(ValueError):
        S.Solver(type="momentum", momentum=-0.1)


class _Stub(S.Trainer):
    """Trainer's checkpoint methods over CPU tensors with the optimizer's state as a dict (no kernel runs)."""

    def __init__(self, tp, solver):
        self.tp, self.global_step, self.solver = tp, 0, solver
        tp.flat_params()
        n = tp.param_flat.numel()
        o = type("O", (), {})()
        o.param = tp.param_flat
        if solver.type == "adam":
            o.sd = {"m": np.zeros(n, F), "v": np.zeros(n, F), "global_step": 0, "beta1_power": F(0.9), "beta2_power": F(0.999)}
        else:
            o.sd = {"accum": np.zeros(n, F), "global_step": 0}
        o.state_dict = lambda: o.sd
        o.load_state_dict = lambda sd: setattr(o, "sd", sd)
        self.optimizer = o


def _layer1_model(pkg, seed):
    arch = [spec for spec in pkg.config.ARCH_3DSSD][:2]
    return pkg.params.init_params(arch, 1, seed=seed, random_bias=True)


def test_checkpoints_hold_slots_of_the_trained_variables_only(pkg, tmp_path):
    d = _layer1_model(pkg, 4)
    rng = np.random.default_rng(1)
    mom = S.Solver(type="momentum")
    a = _Stub(pkg.params.TrainableParams(d, "cpu", trainable=["layer2"]), mom)
    n = a.tp.param_flat.numel()
    a.optimizer.sd = {"accum": rng.standard_normal(n).astype(F), "global_step": 12}
    path = str(tmp_path / "m.npz")
    a.save(path)
    with np.load(path) as z:
        files = set(z.files)
    trained = [k for k, _ in a.tp.named_parameters()]
    assert trained and all(k.startswith("layer2/") for k in trained)
    assert files == set(d) | {k + "/Momentum" for k in trained} | {"global_step"}
    assert not any(k.endswith(("/Adam", "/Adam_1")) for k in files) and "beta1_power" not in files
    with np.load(path) as z:
        assert set(pkg.kitti_io.params_from_tf_variables({k: z[k] for k in z.files})) == set(d)

    b = _Stub(pkg.params.TrainableParams(_layer1_model(pkg, 9), "cpu", trainable=["layer2"]), mom)
    b.load(path)
    assert b.global_step == 12 and b.optimizer.sd["global_step"] == 12
    np.testing.assert_array_equal(b.optimizer.sd["accum"], a.optimizer.sd["accum"])
    for k, t in a.tp.tensors.items():
        assert torch.equal(b.tp.tensors[k], t), k

    wider = _Stub(pkg.params.TrainableParams(_layer1_model(pkg, 9), "cpu", trainable=["layer1", "layer2"]), mom)
    first = [k for k, _ in wider.tp.named_parameters()][0]
    with pytest.raises(ValueError, match=re.escape(first + "/Momentum")):       # the trained set grew: slots are missing
        wider.load(path)
    adam = _Stub(pkg.params.TrainableParams(_layer1_model(pkg, 9), "cpu", trainable=["layer2"]), S.Solver())
    with pytest.raises(ValueError, match=re.escape(trained[0] + "/Adam") + ".*Momentum"):   # another optimizer's slots
        adam.load(path)

    c = _Stub(pkg.params.TrainableParams(_layer1_model(pkg, 9), "cpu", trainable=["layer2"]), S.Solver())
    c.optimizer.sd.update(m=rng.standard_normal(n).astype(F), global_step=5)
    path2 = str(tmp_path / "a.npz")
    c.save(path2)
    with np.load(path2) as z:
        assert set(z.files) == set(d) | {k + s for k in trained for s in ("/Adam", "/Adam_1")} | set(S.SCALARS)
    with pytest.raises(ValueError, match=re.escape(trained[0] + "/Momentum") + ".*Adam"):
        _Stub(pkg.params.TrainableParams(_layer1_model(pkg, 9), "cpu", trainable=["layer2"]), mom).load(path2)
    narrower = _Stub(pkg.params.TrainableParams(_layer1_model(pkg, 9), "cpu", trainable=["layer2/conv0"]), S.Solver())
    narrower.load(path2)                                  # slots of more variables than trained: the trained ones are there
    np.testing.assert_array_equal(narrower.optimizer.sd["m"], c.optimizer.sd["m"][:narrower.tp.param_flat.numel()])


def test_exchange_sizes_follow_the_trained_set(pkg):
    """DataParallel's symmetric memory is sized by the trained gradient alone: the allreduce of the frozen-below set is
    the layout of its own element count, smaller than the full model's."""
    D = pkg.dist
    d = model(pkg)
    full = pkg.params.TrainableParams(d, "cpu")
    top = pkg.params.TrainableParams(d, "cpu", trainable=TOP)
    n = sum(t.numel() for t in top.parameters())
    assert n == sum(d[k].size for k in pkg.params.trained_names(_trainables(d), TOP))
    for world in (1, 2, 8):
        got = D.DataParallel.symmetric_bytes(top, world, 16)
        assert got < D.DataParallel.symmetric_bytes(full, world, 16)
        assert got - D.DataParallel.symmetric_bytes(full, world, 16) == \
            D._round(D.allreduce_layout(n, world, 16).nbytes, 256) - \
            D._round(D.allreduce_layout(sum(t.numel() for t in full.parameters()), world, 16).nbytes, 256)
