"""Backward kernels of the training path on the GPU (-m gpu): each kernel against numpy / float64, the differentiable
layers against the teacher-forced float64 restatement of tests/test_train_grad_cpu.py, the forward of the trainable path
against the non-trainable training path, and one training step of the scaled backbone + head."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from test_backbone_gpu import compact_scene, rel_err, scaled_arch
from test_train_grad_cpu import compare_grads, run_sa, run_vote_cg, sa_case, vote_cg_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _time_train():
    spec = importlib.util.spec_from_file_location("time_train", os.path.join(ROOT, "tools", "time_train.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def rowgroup_max_grad_f32(y, g, cnt=None):
    """float32 numpy restatement of rowgroup_max_grad: y (groups, pool, c), g (groups, c), cnt (groups,) or None ->
    (ind / num) * (g * mask), TF's _MinOrMaxGrad after the Mul gradient of the mask, in the kernel's operation order."""
    ind = (y == y.max(axis=1, keepdims=True)).astype(np.float32)
    num = ind.sum(axis=1, keepdims=True).astype(np.float32)
    gm = g * (cnt > 0).astype(np.float32)[:, None] if cnt is not None else g
    return ((ind / num) * gm[:, None, :]).astype(np.float32)


def test_rowgroup_max_grad_bit_exact_with_ties_and_empty_groups(pkg, cuda):
    rng = np.random.default_rng(0)
    groups, pool, c = 300, 16, 40
    y = rng.integers(-3, 4, (groups, pool, c)).astype(np.float32) * np.float32(0.5)     # many exact ties
    y[::7, 3:] = y[::7, :1]                                                              # back-filled neighbour lists
    cnt = rng.integers(0, 5, groups).astype(np.int32)
    cnt[::5] = 0
    g = rng.standard_normal((groups, c)).astype(np.float32)
    got = pkg.tf_ops.rowgroup_max_grad(torch.from_numpy(y).to(cuda), torch.from_numpy(g).to(cuda), pool,
                                       torch.from_numpy(cnt).to(cuda)).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), rowgroup_max_grad_f32(y, g, cnt).view(np.uint32))


def test_vote_translate_grad_bit_exact_at_bounds(pkg, cuda):
    rng = np.random.default_rng(1)
    lo = np.array([-3.0, -3.0, -2.0], np.float32)
    off = rng.uniform(-4, 4, (2, 500, 3)).astype(np.float32)
    off[0, :50] = lo
    off[0, 50:100] = -lo
    off[1, :20] = np.nextafter(lo, np.float32(-10))
    g = rng.standard_normal((2, 500, 3)).astype(np.float32)
    got = pkg.tf_ops.vote_translate_grad(torch.from_numpy(off).to(cuda), torch.from_numpy(g).to(cuda), lo).cpu().numpy()
    exp = np.where((off >= lo) & (off <= -lo), g, np.float32(0))
    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))


@pytest.mark.parametrize("relu", [True, False])
def test_bn_train_grad_vs_float64(pkg, cuda, relu):
    rng = np.random.default_rng(2)
    rows, c = 20011, 67
    x = (rng.standard_normal((rows, c)) * 2 + 0.5).astype(np.float32)
    gamma = rng.uniform(0.5, 1.5, c).astype(np.float32)
    beta = (0.1 * rng.standard_normal(c)).astype(np.float32)
    go = rng.standard_normal((rows, c)).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(cuda)
    _, scale, shift, mean, var = pkg.tf_ops.bn_train(t(x), t(gamma), t(beta), relu=relu)
    gx, gg, gb = pkg.tf_ops.bn_train_grad(t(x), t(go), scale, shift, mean, var, t(gamma), relu=relu)
    sc, sh, mu, va = (a.cpu().numpy().astype(np.float64) for a in (scale, shift, mean, var))
    g = go.astype(np.float64)
    if relu:
        g = g * ((torch.from_numpy(x).to(cuda) * scale + shift).cpu().numpy() > 0)   # the forward's own decision
    r = 1.0 / np.sqrt(va + 1e-3)
    xh = (x.astype(np.float64) - mu) * r
    sg, sgx = g.sum(0), (g * xh).sum(0)
    egx = gamma.astype(np.float64) * r / rows * (rows * g - sg - xh * sgx)
    for got, exp in ((gx, egx), (gg, sgx), (gb, sg)):
        got = got.cpu().numpy().astype(np.float64)
        assert np.abs(got - exp).max() <= 1e-5 * np.abs(exp).max()


def _arch_shapes(pkg):
    d = pkg.params.init_params(pkg.config.ARCH_3DSSD, 1)
    d.update(pkg.params.init_head_params(512))
    return sorted({v.shape for k, v in d.items() if k.endswith("/weights")})


def test_linear_wgrad_every_arch_shape_vs_float64(pkg, cuda):
    shapes = _arch_shapes(pkg)
    assert (4, 32) in shapes and any(ci in (67, 131, 259) for ci, _ in shapes) and any(ci == 1536 for ci, _ in shapes)
    rng = np.random.default_rng(3)
    for cin, cout in shapes:
        for rows in (1, 777, 4099):
            x = torch.from_numpy(rng.standard_normal((rows, cin)).astype(np.float32)).to(cuda)
            dz = torch.from_numpy(rng.standard_normal((rows, cout)).astype(np.float32)).to(cuda)
            gw, gb = pkg.tf_ops.linear_wgrad(x, dz)
            ew = (x.double().t() @ dz.double()).cpu().numpy()
            eb = dz.double().sum(0).cpu().numpy()
            assert rel_err(gw.cpu().numpy(), ew) <= 1e-4, (cin, cout, rows)
            assert rel_err(gb.cpu().numpy(), eb) <= 1e-6, (cin, cout, rows)


def test_linear_wgrad_two_million_rows_deterministic(pkg, cuda):
    g = torch.Generator(device=cuda).manual_seed(4)
    rows = 2 * 1024 * 1024 + 37
    x = torch.randn((rows, 4), device=cuda, generator=g)
    dz = torch.randn((rows, 32), device=cuda, generator=g) * 1e-3
    gw, gb = pkg.tf_ops.linear_wgrad(x, dz)
    gw2, gb2 = pkg.tf_ops.linear_wgrad(x, dz)
    assert torch.equal(gw, gw2) and torch.equal(gb, gb2)
    ew = (x.double().t() @ dz.double()).cpu().numpy()
    assert rel_err(gw.cpu().numpy(), ew) <= 1e-4
    x = torch.randn((300001, 259), device=cuda, generator=g)
    dz = torch.randn((300001, 256), device=cuda, generator=g)
    a, b = pkg.tf_ops.linear_wgrad(x, dz)
    assert torch.equal(a, pkg.tf_ops.linear_wgrad(x, dz)[0])
    assert rel_err(a.cpu().numpy(), (x.double().t() @ dz.double()).cpu().numpy()) <= 1e-4


def test_group_concat_grad_vs_float64(pkg, cuda):
    rng = np.random.default_rng(5)
    b, n, c, m, ns = 2, 300, 13, 40, 16
    idx = rng.integers(0, n, (b, m, ns)).astype(np.int32)
    idx[:, :, 8:] = idx[:, :, :1]
    gx = rng.standard_normal((b, m, ns, c + 3)).astype(np.float32)
    gp, gxyz, gnew = pkg.tf_ops.group_concat_grad(torch.from_numpy(gx).to(cuda), torch.from_numpy(idx).to(cuda), n, c)
    ep, exyz = np.zeros((b, n, c)), np.zeros((b, n, 3))
    for s in range(b):
        np.add.at(ep[s], idx[s].reshape(-1), gx[s, ..., :c].reshape(-1, c).astype(np.float64))
        np.add.at(exyz[s], idx[s].reshape(-1), gx[s, ..., c:].reshape(-1, 3).astype(np.float64))
    enew = -gx[..., c:].astype(np.float64).sum(2)
    for got, exp in ((gp, ep), (gxyz, exyz), (gnew, enew)):
        assert np.abs(got.cpu().numpy() - exp).max() <= 1e-6 * np.abs(exp).max()


def test_trainable_forward_bit_identical_to_prepared(pkg, cuda):
    xyz, feats, d, args = sa_case(pkg, seed=9, n=1024)
    x, f = torch.from_numpy(xyz).to(cuda), torch.from_numpy(feats).to(cuda)
    pp = pkg.params.prepare({k: v.copy() for k, v in d.items()}, cuda)
    tp = pkg.params.TrainableParams(d, cuda)
    a = pkg.pointnet_sa_module_msg(x, f, *args, aggregation_channel=24, params=pp)[1]
    b = pkg.pointnet_sa_module_msg(x, f, *args, aggregation_channel=24, params=tp)[1]
    assert torch.equal(a, b.detach())
    for k, t in tp.tensors.items():
        if k.endswith(("moving_mean", "moving_variance")):
            scope, name = k.rsplit("/bn/", 1)
            assert torch.equal(pp.bn_state(scope)[name], t), k


def test_sa_layer_gradients_teacher_forced(pkg, cuda):
    xyz, feats, d, args = sa_case(pkg, seed=10, n=1024)
    tp, P, dbg, extra, _ = run_sa(pkg, xyz, feats, d, args, cuda)
    compare_grads(tp, P, extra=extra)


def test_vote_to_cg_gradients_teacher_forced(pkg, cuda):
    xyz, feats, d, args = vote_cg_case(pkg, seed=11, n=256)
    tp, P, extra, _ = run_vote_cg(pkg, xyz, feats, d, args, cuda)
    assert tp.grads()["vote/vote_layer_0/weights"].abs().max() > 0
    compare_grads(tp, P, extra=extra)


def test_scaled_backbone_and_head_training_step(pkg, cuda):
    tt = _time_train()
    arch = scaled_arch(pkg, 8)
    tp = tt.trainable(arch, cuda, seed=4)
    pts = torch.from_numpy(compact_scene(2, 2048, seed=40)).to(cuda)
    xyz, feat = pkg.tf_ops.split_points(pts)
    loss0 = tt.step(arch, tp, xyz, feat)
    for k, g in tp.grads().items():
        assert g is not None and torch.isfinite(g).all(), k
        if k.endswith("/weights"):
            assert g.abs().max() > 0, k
    # Adam's first step moves every parameter by about lr * sign(grad): to first order the loss drops by lr * sum|grad|
    lr = 1e-5
    predicted = lr * sum(g.abs().sum().item() for g in tp.grads().values())
    opt = torch.optim.Adam(tp.parameters(), lr=lr)
    opt.step()
    with torch.no_grad():
        outs, offs = tt.train_forward(arch, tp, xyz, feat)
        loss1 = sum((o ** 2).mean() for o in outs) + sum((o ** 2).mean() for o in offs)
    drop = loss0.item() - loss1.item()
    assert drop > 0 and 0.3 < drop / predicted < 3.0, (loss0.item(), loss1.item(), predicted)
