"""CPU dry run of the differentiable training path (params.TrainableParams with is_training=True): the forward kernels
are replaced by the CPU stand-ins of test_orchestration_cpu's `dry` fixture, the backward kernels by float64 torch lines,
and the gradients of a random linear functional of the outputs are compared with torch.autograd in float64 over a
literal restatement of the TF op sequence (layers_util.py / tf_util.py).  The restatement takes its ReLU masks and
max-pool indicator sets from the path's own forward ("teacher-forced"), so rounding near a decision cannot move a
row's gradient; what is left to disagree is wiring: a wrong column slice, a missing mask, a missing new_xyz path.
The reference functions here are shared with tests/test_train_grad_gpu.py."""
import numpy as np
import pytest
import torch

from test_orchestration_cpu import dry  # noqa: F401  (fixture)

EPS = 1e-3


# ---- float64 restatement of the TF graph, decisions from the path under test --------------------------------------

class Recording:
    """Wraps a TrainableParams so that every conv records its (pre-BN, post-activation) tensors by scope."""

    def __init__(self, tp):
        self.tp, self.rec = tp, {}

    def conv_train(self, scope, x, bn=True, bn_decay=None, relu=True, debug=None):
        self.rec[scope] = []
        out = self.tp.__class__.conv_train(self.tp, scope, x, bn, bn_decay, relu, self.rec[scope])
        if debug is not None:
            debug.extend(self.rec[scope])
        return out


def recording(pkg, tp):
    rec = Recording(tp)
    tp.conv_train = rec.conv_train          # instance attribute: layers call params.conv_train(...)
    return rec.rec


def ref_leaves(tp):
    return {k: t.detach().double().cpu().clone().requires_grad_(True) for k, t in tp.named_parameters()}


def ref_conv(P, rec, scope, x, bn, relu):
    """tf_util.conv1d/conv2d + batch_norm_template(is_training=True) + ReLU with the path's ReLU mask."""
    z = x @ P[scope + "/weights"] + P[scope + "/biases"]
    if bn:
        flat = z.reshape(-1, z.shape[-1])
        mean = flat.mean(0)
        var = ((flat - mean) ** 2).mean(0)                         # tf.nn.moments: population variance
        z = (z - mean) / torch.sqrt(var + EPS) * P[scope + "/bn/gamma"] + P[scope + "/bn/beta"]
    if relu:
        post = rec[scope][0][1].detach().double().cpu()
        z = z * (post > 0).to(z.dtype)                             # ReluGrad: where the output is > 0
    return z


def ref_group_max(g, post, cnt):
    """tf.reduce_max(axis=2) * mask with the path's indicator set: (ind / num) * value summed = the max, and its
    gradient is TF's even split among tied maxima."""
    post = post.detach().double().cpu()
    ind = (post == post.amax(dim=-2, keepdim=True)).to(g.dtype)
    pooled = (g * ind / ind.sum(dim=-2, keepdim=True)).sum(dim=-2)
    return pooled * (cnt.cpu() > 0).to(g.dtype).unsqueeze(-1)


def gather_rows(src, idx):
    idx = idx.long().cpu()
    return src[torch.arange(src.shape[0]).view(-1, 1, *([1] * (idx.dim() - 2))), idx]


def ref_sa_msg(P, rec, xyz, points, new_xyz, idx_list, cnt_list, mlp_list, scope, use_agg):
    outs = []
    for i, (idx, cnt) in enumerate(zip(idx_list, cnt_list)):
        g = torch.cat([gather_rows(points, idx), gather_rows(xyz, idx) - new_xyz.unsqueeze(2)], -1)   # :160-165
        for j in range(len(mlp_list[i])):
            g = ref_conv(P, rec, "%s/conv%d_%d" % (scope, i, j), g, True, True)
        last = "%s/conv%d_%d" % (scope, i, len(mlp_list[i]) - 1)
        outs.append(ref_group_max(g, rec[last][0][1], cnt))
    out = torch.cat(outs, -1)
    return ref_conv(P, rec, scope + "/ensemble", out, True, True) if use_agg else out


def ref_vote(P, rec, xyz, points, nl, scope, rng):
    for i in range(nl):
        points = ref_conv(P, rec, "%s/vote_layer_%d" % (scope, i), points, True, True)
    off = ref_conv(P, rec, scope + "/vote_offsets", points, False, False)
    lo = torch.tensor(rng, dtype=off.dtype)
    inside = ((off >= lo) & (off <= -lo)).to(off.dtype)             # tf.maximum / tf.minimum: ties go to the offset
    clamped = off * inside + torch.minimum(torch.maximum(off, lo), -lo).detach() * (1 - inside)
    return xyz + clamped, points, off


def ref_head(P, rec, feat):
    cls = ref_conv(P, rec, "pred_cls", ref_conv(P, rec, "pred_cls_base", feat, True, True), False, False)
    reg = ref_conv(P, rec, "pred_reg", ref_conv(P, rec, "pred_reg_base", feat, True, True), False, False)
    return cls, reg


def compare_grads(tp, P, tol=1e-3, extra=()):
    """Every trainable tensor's gradient against the float64 reference (global-norm relative error); biases of convs
    followed by batch-statistics BatchNorm have a true gradient of 0 and get an absolute bound instead."""
    got = tp.grads()
    for k, t in P.items():
        g = got[k]
        assert g is not None and torch.isfinite(g).all(), k
        g = g.detach().double().cpu()
        scope = k.rsplit("/", 1)[0]
        if k.endswith("/biases") and (scope + "/bn/gamma") in P:
            gw = got[scope + "/weights"].detach().abs().max().item()
            assert g.abs().max().item() <= 1e-5 * gw, (k, g.abs().max().item(), gw)
            continue
        e = t.grad
        # floor: a tensor whose true gradient cancels (beta of a channel whose shift the next BatchNorm removes) is held
        # to the scale of its layer's weight gradient
        layer = scope[:-3] if scope.endswith("/bn") else scope
        scale = max(e.abs().max().item(), 1e-2 * P[layer + "/weights"].grad.abs().max().item(), 1e-30)
        assert (g - e).abs().max().item() <= tol * scale, (k, (g - e).abs().max().item() / scale)
    for name, g, e in extra:
        g, e = g.detach().double().cpu(), e.detach().double()
        scale = max(e.abs().max().item(), 1e-30)
        assert (g - e).abs().max().item() <= tol * scale, (name, (g - e).abs().max().item() / scale)


def conv_params(pkg, rng, d, scope, cin, cout, bn):
    pkg.params._conv_init(rng, d, scope, cin, cout, bn)
    d[scope + "/biases"] = (0.1 * rng.standard_normal(cout)).astype(np.float32)


def sa_case(pkg, seed=0, c=8, n=256, dev="cpu"):
    """One SA layer with fusion sampling (F-FPS + D-FPS), two scales and aggregation (3DSSD layer-2 shaped, small)."""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(0, 2, (2, n, 3)).astype(np.float32)
    feats = rng.standard_normal((2, n, c)).astype(np.float32)
    mlp = [[8, 16], [8, 16]]
    d = {}
    for i, m in enumerate(mlp):
        cin = c + 3
        for j, co in enumerate(m):
            conv_params(pkg, rng, d, "sa/conv%d_%d" % (i, j), cin, co, True)
            cin = co
    conv_params(pkg, rng, d, "sa/ensemble", 32, 24, True)
    args = ([0.4, 0.8], [16, 32], mlp, True, None, True, [-1], ["FS"], [32], None, False, "sa", False)
    return xyz, feats, d, args


def run_sa(pkg, xyz, feats, d, args, dev):
    tp = pkg.params.TrainableParams(d, dev)
    rec = recording(pkg, tp)
    x = torch.from_numpy(xyz).to(dev).requires_grad_(True)
    f = torch.from_numpy(feats).to(dev).requires_grad_(True)
    new_xyz, out, fps_idx, dbg = pkg.pointnet_sa_module_msg(x, f, *args, aggregation_channel=24, params=tp, return_debug=True)
    R = torch.from_numpy(np.random.default_rng(7).standard_normal(tuple(out.shape)).astype(np.float32)).to(dev)
    (out * R).sum().backward()
    P = ref_leaves(tp)
    xr = torch.from_numpy(xyz).double().requires_grad_(True)
    fr = torch.from_numpy(feats).double().requires_grad_(True)
    nx = gather_rows(xr, fps_idx)
    exp = ref_sa_msg(P, rec, xr, fr, nx, dbg["idx"], dbg["cnt"], args[2], "sa", True)
    (exp * R.double().cpu()).sum().backward()
    return tp, P, dbg, [("xyz", x.grad, xr.grad), ("features", f.grad, fr.grad)], (out, exp)


def vote_cg_case(pkg, seed=1, c=16, n=64):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(0, 3, (2, n, 3)).astype(np.float32)
    feats = rng.standard_normal((2, n, c)).astype(np.float32)
    d = {}
    conv_params(pkg, rng, d, "vote/vote_layer_0", c, 16, True)
    conv_params(pkg, rng, d, "vote/vote_offsets", 16, 3, False)
    d["vote/vote_offsets/weights"] *= 4.0                         # some offsets land beyond the clamp
    for i in range(2):
        conv_params(pkg, rng, d, "cg/conv%d_0" % i, c + 3, 16, True)
    conv_params(pkg, rng, d, "cg/ensemble", 32, 24, True)
    args = ([0.8, 1.6], [16, 32], [[16], [16]], True, None, True, [-1], ["D-FPS"], [n], None, False, "cg", False)
    return xyz, feats, d, args


def run_vote_cg(pkg, xyz, feats, d, args, dev, rng_clamp=(-1.0, -1.0, -0.5)):
    tp = pkg.params.TrainableParams(d, dev)
    rec = recording(pkg, tp)
    x = torch.from_numpy(xyz).to(dev).requires_grad_(True)
    f = torch.from_numpy(feats).to(dev).requires_grad_(True)
    ctr, _, off = pkg.vote_layer(x, f, [16], True, None, True, "vote", params=tp, max_translate_range=list(rng_clamp))
    _, out, fps_idx, dbg = pkg.pointnet_sa_module_msg(x, f, *args, vote_ctr=ctr, aggregation_channel=24, params=tp, return_debug=True)
    rs = np.random.default_rng(8)
    R = torch.from_numpy(rs.standard_normal(tuple(out.shape)).astype(np.float32)).to(dev)
    Ro = torch.from_numpy(rs.standard_normal(tuple(off.shape)).astype(np.float32)).to(dev)
    ((out * R).sum() + (off * Ro).sum()).backward()            # the raw offsets feed the vote loss
    P = ref_leaves(tp)
    xr = torch.from_numpy(xyz).double().requires_grad_(True)
    fr = torch.from_numpy(feats).double().requires_grad_(True)
    ctr_r, _, off_r = ref_vote(P, rec, xr, fr, 1, "vote", rng_clamp)
    exp = ref_sa_msg(P, rec, xr, fr, gather_rows(ctr_r, fps_idx), dbg["idx"], dbg["cnt"], args[2], "cg", True)
    ((exp * R.double().cpu()).sum() + (off_r * Ro.double().cpu()).sum()).backward()
    return tp, P, [("xyz", x.grad, xr.grad), ("features", f.grad, fr.grad)], off


# ---- the dry fixture: float64 stand-ins of the training kernels ------------------------------------------------------

@pytest.fixture()
def gdry(dry, monkeypatch):
    pkg = dry
    T = pkg.tf_ops

    def bn_train(x, gamma, beta, moving_mean=None, moving_var=None, decay=0.9, relu=True, eps=EPS):
        flat = x.reshape(-1, x.shape[-1]).double()
        mean = flat.mean(0)
        var = ((flat - mean) ** 2).mean(0)
        inv = gamma.double() / torch.sqrt(var + eps)
        scale, shift = inv.float(), (beta.double() - mean * inv).float()
        y = x * scale + shift
        if moving_mean is not None:
            moving_mean.sub_(((moving_mean.double() - mean) * (1.0 - decay)).float())
            moving_var.sub_(((moving_var.double() - var) * (1.0 - decay)).float())
        return (torch.relu(y) if relu else y), scale, shift, mean.float(), var.float()

    def bn_train_grad(x, g, scale, shift, mean, var, gamma, relu=True, eps=EPS):
        c = x.shape[-1]
        x2, g2 = x.reshape(-1, c).double(), g.reshape(-1, c).double()
        if relu:
            g2 = g2 * ((x.reshape(-1, c) * scale + shift) > 0).double()
        r = 1.0 / torch.sqrt(var.double() + eps)
        xh = (x2 - mean.double()) * r
        sg, sgx, nn = g2.sum(0), (g2 * xh).sum(0), x2.shape[0]
        gx = gamma.double() * r / nn * (nn * g2 - sg - xh * sgx)
        return gx.float().reshape(x.shape), sgx.float(), sg.float()

    def linear_wgrad(x, dz, want_bias=True):
        a, b = x.reshape(-1, x.shape[-1]).double(), dz.reshape(-1, dz.shape[-1]).double()
        return (a.t() @ b).float(), (b.sum(0).float() if want_bias else None)

    def rowgroup_max(y, pool, rowmask=None):
        out = y.max(dim=-2).values
        return out * (rowmask > 0).unsqueeze(-1).to(out.dtype) if rowmask is not None else out

    def rowgroup_max_grad(y, g, pool, rowmask=None):
        ind = (y == y.amax(dim=-2, keepdim=True)).float()
        gm = g * (rowmask > 0).float().unsqueeze(-1) if rowmask is not None else g
        return (ind / ind.sum(dim=-2, keepdim=True)) * gm.unsqueeze(-2)

    def group_concat_grad(gx, idx, n, c, want_points=True, want_xyz=True, want_new_xyz=True):
        b = gx.shape[0]
        flat_idx = (idx.long() + torch.arange(b).view(b, 1, 1) * n).reshape(-1)
        rows = gx.reshape(-1, gx.shape[-1]).double()
        gp = torch.zeros(b * n, c, dtype=torch.float64).index_add_(0, flat_idx, rows[:, :c]).float().view(b, n, c) if (want_points and c) else None
        gxyz = torch.zeros(b * n, 3, dtype=torch.float64).index_add_(0, flat_idx, rows[:, c:c + 3]).float().view(b, n, 3) if want_xyz else None
        gnew = -gx[..., c:c + 3].double().sum(2).float() if want_new_xyz else None
        return gp, gxyz, gnew

    def vote_translate_grad(off, g, rng):
        lo = torch.tensor(rng, dtype=off.dtype)
        return torch.where((off[..., :3] >= lo) & (off[..., :3] <= -lo), g, torch.zeros_like(g))

    for k, v in dict(bn_train=bn_train, bn_train_grad=bn_train_grad, linear_wgrad=linear_wgrad, rowgroup_max=rowgroup_max,
                     rowgroup_max_grad=rowgroup_max_grad, group_concat_grad=group_concat_grad,
                     vote_translate_grad=vote_translate_grad, gather_point=gather_rows).items():
        monkeypatch.setattr(T, k, v)
    return pkg


def test_sa_layer_fusion_sampling_aggregation_gradients(gdry):
    pkg = gdry
    xyz, feats, d, args = sa_case(pkg)
    tp, P, dbg, extra, _ = run_sa(pkg, xyz, feats, d, args, "cpu")
    assert any((c < 16).any() for c in dbg["cnt"])                  # back-filled neighbour lists: ties in the max-pool
    assert len(dbg["convs"]) == 5                                    # return_debug carries every conv's tensors
    compare_grads(tp, P, extra=extra)


def test_vote_layer_to_cg_layer_gradients(gdry):
    pkg = gdry
    xyz, feats, d, args = vote_cg_case(pkg)
    tp, P, extra, off = run_vote_cg(pkg, xyz, feats, d, args, "cpu")
    lim = torch.tensor([1.0, 1.0, 0.5])
    assert (off.detach().abs() > lim).any() and (off.detach().abs() < lim).any()
    # the CG features reach the vote layer only through new_xyz = vote centres
    g = tp.grads()["vote/vote_layer_0/weights"]
    assert g is not None and g.abs().max() > 0
    compare_grads(tp, P, extra=extra)


def test_head_gradients(gdry):
    pkg = gdry
    rng = np.random.default_rng(2)
    feat = np.maximum(rng.standard_normal((2, 48, 32)), 0).astype(np.float32)
    tp = pkg.params.TrainableParams(pkg.params.init_head_params(32, mlp=(), seed=3), "cpu")
    rec = recording(pkg, tp)
    f = torch.from_numpy(feat).requires_grad_(True)
    out = pkg.head.box_regression_head(f, 1, 1, 6, True, True, params=tp)
    R = [torch.from_numpy(rng.standard_normal(tuple(o.shape)).astype(np.float32)) for o in out]
    sum((o * r).sum() for o, r in zip(out, R)).backward()
    P = ref_leaves(tp)
    fr = torch.from_numpy(feat).double().requires_grad_(True)
    cls, reg = ref_head(P, rec, fr)
    reg = reg.view(2, 48, 1, 30)
    exp = (cls, reg[..., :6], reg[..., 6:18], reg[..., 18:])
    sum((e * r.double()).sum() for e, r in zip(exp, R)).backward()
    compare_grads(tp, P, extra=[("features", f.grad, fr.grad)])


def test_reduce_max_ties_split_evenly(gdry):
    """Two and three equal maxima share the gradient evenly; a masked group gets none (the TF rule the kernel restates)."""
    T = gdry.tf_ops
    y = torch.tensor([[[1.0, 5.0], [3.0, 5.0], [3.0, 2.0], [0.0, 5.0]],
                      [[7.0, 1.0], [7.0, 1.0], [7.0, 1.0], [6.0, 0.0]],
                      [[1.0, 1.0], [2.0, 2.0], [3.0, 3.0], [4.0, 4.0]]]).requires_grad_(True)
    cnt = torch.tensor([4, 2, 0], dtype=torch.int32)
    out = T.group_max_train(y, 4, cnt)
    assert out.tolist() == [[3.0, 5.0], [7.0, 1.0], [0.0, 0.0]]
    out.backward(torch.tensor([[6.0, 3.0], [3.0, 9.0], [1.0, 1.0]]))
    assert y.grad.tolist() == [[[0.0, 1.0], [3.0, 1.0], [3.0, 0.0], [0.0, 1.0]],
                               [[1.0, 3.0], [1.0, 3.0], [1.0, 3.0], [0.0, 0.0]],
                               [[0.0, 0.0], [0.0, 0.0], [0.0, 0.0], [0.0, 0.0]]]


def test_vote_clamp_bounds_are_inclusive(gdry):
    T = gdry.tf_ops
    off = torch.tensor([[[-1.0, 1.0, 0.5], [-1.0001, 1.0001, -0.5], [0.0, -0.25, 0.75]]]).requires_grad_(True)
    xyz = torch.zeros((1, 3, 3), requires_grad=True)
    out = T.vote_translate_train(xyz, off, (-1.0, -1.0, -0.5))
    out.backward(torch.full((1, 3, 3), 2.0))
    assert off.grad.tolist() == [[[2.0, 2.0, 2.0], [0.0, 0.0, 2.0], [2.0, 2.0, 0.0]]]
    assert xyz.grad.tolist() == [[[2.0] * 3] * 3]


def test_trainable_params_round_trip(gdry, oracle_ops):
    pkg = gdry
    from oracle import layers as olayers
    xyz, feats, d, args = sa_case(pkg, seed=5)
    tp = pkg.params.TrainableParams(d, "cpu")
    assert {k: tuple(v.shape) for k, v in tp.tensors.items()} == {k: v.shape for k, v in d.items()}
    names = {k for k, _ in tp.named_parameters()}
    assert names == {k for k in d if not k.endswith(("moving_mean", "moving_variance"))}
    assert all(t.requires_grad for t in tp.parameters())
    x, f = torch.from_numpy(xyz), torch.from_numpy(feats)
    out1 = pkg.pointnet_sa_module_msg(x, f, *args, aggregation_channel=24, params=tp)[1]
    assert not np.array_equal(tp.to_params()["sa/conv0_0/bn/moving_mean"], d["sa/conv0_0/bn/moving_mean"])  # updated in place
    opt = torch.optim.Adam(tp.parameters(), lr=1e-2)
    (out1 ** 2).sum().backward()
    opt.step()
    out2 = pkg.pointnet_sa_module_msg(x, f, *args, aggregation_channel=24, params=tp)[1]
    assert (out2 - out1).abs().max() > 1e-3                          # the step is visible to the next forward
    trained = tp.to_params()
    assert not np.array_equal(trained["sa/conv0_0/weights"], d["sa/conv0_0/weights"])
    args_inf = args[:3] + (False,) + args[4:]
    got = pkg.pointnet_sa_module_msg(x, f, *args_inf, aggregation_channel=24, params=pkg.params.prepare(trained, "cpu"))[1]
    via_tp = pkg.pointnet_sa_module_msg(x, f, *args_inf, aggregation_channel=24, params=tp)[1]
    exp = olayers.pointnet_sa_module_msg(xyz, feats, *args_inf, aggregation_channel=24, params=trained)[1]
    assert torch.equal(got, via_tp)
    assert np.abs(got.numpy() - exp).max() <= 1e-4 * np.abs(exp).max()


def test_inference_dict_and_head_without_trainable_params_unchanged(gdry):
    pkg = gdry
    with pytest.raises(NotImplementedError):
        pkg.head.box_regression_head(torch.zeros((1, 4, 8)), 1, 1, 6, True, True, params=pkg.params.init_head_params(8))
