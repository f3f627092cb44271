"""Weights of the SA path: initialisation in the reference's variable layout and inference-time folding.

Variable names follow the reference's TF scopes (SURVEY.md section 5; lib/utils/layers_util.py:175,185 and
lib/utils/tf_util.py:96,111,119):
  <scope>/conv{i}_{j}/weights [cin,cout]   (TF kernel [1,1,cin,cout] squeezed)
  <scope>/conv{i}_{j}/biases  [cout]
  <scope>/conv{i}_{j}/bn/{gamma,beta,moving_mean,moving_variance} [cout]
  <scope>/ensemble/...                      aggregation conv1d
  <scope>/vote_layer_{i}/..., <scope>/vote_offsets/...  (vote layer, layers_util.py:18-19)
"""
import numpy as np
import torch

from . import config as _cfg

FUSED_SMEM_LIMIT = 226 * 1024
BN_EPS = 1e-3  # tf.contrib.layers.batch_norm default epsilon (tf_util.py:439-444 does not override it)


def _conv_init(rng, params, scope, cin, cout, bn):
    limit = np.sqrt(6.0 / (cin + cout))  # tf.contrib.layers.xavier_initializer, uniform (tf_util.py:41)
    params[scope + "/weights"] = rng.uniform(-limit, limit, size=(cin, cout)).astype(np.float32)
    params[scope + "/biases"] = np.zeros((cout,), np.float32)  # tf_util.py:110
    if bn:  # randomised statistics so that the folding is actually exercised (SURVEY.md section 8d)
        params[scope + "/bn/gamma"] = rng.uniform(0.5, 1.5, size=(cout,)).astype(np.float32)
        params[scope + "/bn/beta"] = (0.1 * rng.standard_normal(cout)).astype(np.float32)
        params[scope + "/bn/moving_mean"] = (0.1 * rng.standard_normal(cout)).astype(np.float32)
        params[scope + "/bn/moving_variance"] = rng.uniform(0.5, 1.5, size=(cout,)).astype(np.float32)


def init_params(arch, in_channels, seed=0, random_bias=False, aggregation=None):
    """Random weights for every conv of `arch` (numpy dict keyed by TF variable name).  aggregation: as
    config.layer_channels (None: config.AGGREGATION_SA_FEATURE)."""
    aggregation = _cfg.AGGREGATION_SA_FEATURE if aggregation is None else aggregation
    rng = np.random.default_rng(seed)
    params = {}
    ch = _cfg.layer_channels(arch, in_channels, aggregation)
    for li, spec in enumerate(arch):
        (_, feat_i, radius, _, mlps, bn, _, _, _, _, _, ltype, scope, _, _, agg) = spec
        cin = ch[feat_i[0]]
        if ltype == "SA_Layer":
            if len(radius) == 0:
                continue
            for i, mlp in enumerate(mlps):
                c = cin + 3
                for j, cout in enumerate(mlp):
                    _conv_init(rng, params, "%s/conv%d_%d" % (scope, i, j), c, cout, bn)
                    c = cout
            if agg is not None and agg != -1 and aggregation:
                _conv_init(rng, params, scope + "/ensemble", sum(m[-1] for m in mlps), agg, bn)
        elif ltype == "Vote_Layer":
            c = cin
            for i, cout in enumerate(mlps):
                _conv_init(rng, params, "%s/vote_layer_%d" % (scope, i), c, cout, bn)
                c = cout
            _conv_init(rng, params, scope + "/vote_offsets", c, 3, False)
        elif ltype == "SA_Layer_SSG_Last":
            c = cin + 3
            for j, cout in enumerate(mlps):
                _conv_init(rng, params, "%s/conv%d" % (scope, j), c, cout, bn)
                c = cout
        elif ltype == "FP_Layer":
            c = cin + ch[feat_i[1]] if len(feat_i) > 1 else cin
            for j, cout in enumerate(mlps):
                _conv_init(rng, params, "%s/conv_%d" % (scope, j), c, cout, bn)
                c = cout
    if random_bias:
        for k in list(params):
            if k.endswith("/biases"):
                params[k] = (0.1 * rng.standard_normal(params[k].shape)).astype(np.float32)
    return params


def round16(x):
    return (int(x) + 15) // 16 * 16


def init_head_params(cin, mlp=(128,), cls_channels=1, reg_channels=6 + 2 * 12, seed=1, scope=''):
    """Random weights of the detection head (head_builder.py:93-95, head_util.py:26-41) keyed by the reference's
    variable names: conv1d_{i}, pred_cls_base, pred_cls, pred_reg_base, pred_reg (scope '' in 3dssd.yaml:68)."""
    rng = np.random.default_rng(seed)
    pre = "" if scope == "" else scope + "/"
    params = {}
    c = cin
    for i, ch in enumerate(mlp):
        _conv_init(rng, params, "%sconv1d_%d" % (pre, i), c, ch, True)
        c = ch
    _conv_init(rng, params, pre + "pred_cls_base", c, 128, True)
    _conv_init(rng, params, pre + "pred_cls", 128, cls_channels, False)
    _conv_init(rng, params, pre + "pred_reg_base", c, 128, True)
    _conv_init(rng, params, pre + "pred_reg", 128, reg_channels, False)
    for k in list(params):
        if k.endswith("/biases"):
            params[k] = (0.1 * rng.standard_normal(params[k].shape)).astype(np.float32)
    return params


def init_rcnn_params(feat_channels=128, pooler=None, arch=None, head=None, reg_channels=6 * 4 + 4 + 2 * 12, seed=2):
    """Random weights of PointRCNN's second stage keyed by the reference's variable names: <pooler scope>/conv{i} of the
    region pool's info network (align_channel_network, pool_utils.py:5-16; 5 -> 128 at roi_pool/conv0), the stage-2 SA
    layers (rcnn_layer1-3) on the pooled [info conv | RPN feature] channels, and the head (rcnn_head: conv1d_0, 2 softmax
    class channels, Bin-Anchor regression with BIN_CLASS_NUM 6)."""
    pooler = _cfg.POINTS_POOLER_POINTRCNN if pooler is None else pooler
    arch = _cfg.ARCH_POINTRCNN_RCNN if arch is None else arch
    head = _cfg.HEAD_POINTRCNN_RCNN if head is None else head
    rng = np.random.default_rng(seed)
    params = {}
    c = 5                                                   # [canonical xyz | mask | dist]
    for i, cout in enumerate(pooler[2]):
        _conv_init(rng, params, "%s/conv%d" % (pooler[8], i), c, cout, pooler[7])
        c = cout
    # the stage-2 lists start with [proposal centres, pooled points]: the table's indices are one past init_params's
    shifted = [[[i - 1 for i in spec[0]], [i - 1 for i in spec[1]]] + list(spec[2:]) for spec in arch]
    params.update(init_params(shifted, c + feat_channels, seed=seed + 1, aggregation=False))
    cin = _cfg.layer_channels(shifted, c + feat_channels, aggregation=False)[head[1][0] - 1]
    params.update(init_head_params(cin, mlp=tuple(head[3]), cls_channels=2, reg_channels=reg_channels, seed=seed + 2,
                                   scope=head[6]))
    return params


class FoldedConv:
    """One conv+BN layer folded for inference: y = act((x @ w) * scale + shift).
    For the tensor-core path the weight also exists split in two bf16 terms, transposed to K-major:
    b_hi + b_lo ~= w^T, shape [cout, kp] with kp = round16(cin) (zero padded)."""
    __slots__ = ("w", "scale", "shift", "cin", "cout", "kp", "b_hi", "b_lo")

    def __init__(self, w, scale, shift):
        self.w, self.scale, self.shift = w, scale, shift
        self.cin, self.cout = w.shape
        self.kp = round16(self.cin)
        wt = torch.zeros((self.cout, self.kp), dtype=torch.float32, device=w.device)
        wt[:, : self.cin] = w.t()
        self.b_hi = wt.to(torch.bfloat16)                       # round-to-nearest-even, like the device split
        self.b_lo = (wt - self.b_hi.to(torch.float32)).to(torch.bfloat16)

    @classmethod
    def from_operands(cls, w, scale, shift, b_hi, b_lo):
        """A fold whose split operand already exists (b_hi, b_lo [cout, round16(cin)], built from w elsewhere)."""
        f = cls.__new__(cls)
        f.w, f.scale, f.shift, f.b_hi, f.b_lo = w, scale, shift, b_hi, b_lo
        f.cin, f.cout = w.shape
        f.kp = round16(f.cin)
        if tuple(b_hi.shape) != (f.cout, f.kp) or tuple(b_lo.shape) != (f.cout, f.kp):
            raise ValueError("from_operands: operands %s / %s of a [%d, %d] weight" % (tuple(b_hi.shape), tuple(b_lo.shape), f.cin, f.cout))
        return f


OPERAND_TILE = 32             # csrc/solver.cu works on 32 x 32 tiles of a weight


def operand_layout(weights):
    """Where ssd3d_weight_operands finds and puts every conv weight.  weights: [(offset in the flat parameter buffer, cin,
    cout)].  Returns (table, arena_elems, tiles): table int64 [nw, 8] with rows (param offset, cin, cout, fwd_hi, fwd_lo,
    bwd_hi, bwd_lo, tile_start) -- offsets in bf16 elements of one arena, each weight's four blocks back to back: the
    forward operand [cout, round16(cin)] hi then lo, the grad-x operand [cin, round16(cout)] hi then lo.  Every block is a
    multiple of 16 elements, so all start on 16-byte boundaries."""
    table = np.zeros((len(weights), 8), np.int64)
    off = tiles = 0
    for r, (poff, cin, cout) in enumerate(weights):
        fwd, bwd = cout * round16(cin), cin * round16(cout)
        table[r] = (poff, cin, cout, off, off + fwd, off + 2 * fwd, off + 2 * fwd + bwd, tiles)
        off += 2 * fwd + 2 * bwd
        tiles += -(-round16(cin) // OPERAND_TILE) * -(-round16(cout) // OPERAND_TILE)
    return table, off, tiles


def fold(params, scope, bn, device):
    """inv = gamma * rsqrt(var + eps);  y = (xW + b) * inv + (beta - mean * inv)   (tf_util.py:439-444)."""
    w = np.asarray(params[scope + "/weights"], np.float64)
    b = np.asarray(params.get(scope + "/biases", np.zeros(w.shape[1])), np.float64)
    if bn:
        g = np.asarray(params[scope + "/bn/gamma"], np.float64)
        be = np.asarray(params[scope + "/bn/beta"], np.float64)
        mu = np.asarray(params[scope + "/bn/moving_mean"], np.float64)
        var = np.asarray(params[scope + "/bn/moving_variance"], np.float64)
        inv = g / np.sqrt(var + BN_EPS)
        scale, shift = inv, (b - mu) * inv + be
    else:
        scale, shift = np.ones_like(b), b
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(device)
    return FoldedConv(t(w), t(scale), t(shift))


def _k_blocks(kp):
    """Operand layout of the fused kernel for a padded K: (nfull, rbt) = number of 64-wide k-blocks (128-byte rows) and
    the row bytes of the tail block -- 0 / 32 / 64 / 128 for a remainder of 0 / 16 / 32 / 48 columns (must match
    sf_nfull / sf_rbt in csrc/sa_fused.cu)."""
    rem = kp % 64
    return kp // 64, 0 if rem == 0 else (32 if rem <= 16 else (64 if rem <= 32 else 128))


def _swizzle_block(blk, rb):
    """[npad, rb/2] bf16 -> canonical K-major (wgmma / TMA) image with swizzle span rb: 16-byte chunk j of row r is stored at
    chunk j ^ ((r >> log2(128/rb)) & (rb/16 - 1)), i.e. SWIZZLE_128B / _64B / _32B for rb = 128 / 64 / 32."""
    npad = blk.shape[0]
    nc = rb // 16
    sh = {128: 0, 64: 1, 32: 2}[rb]
    t = blk.reshape(npad, nc, 8)
    r = torch.arange(npad, device=blk.device).view(npad, 1, 1)
    j = torch.arange(nc, device=blk.device).view(1, nc, 1)
    src = (j ^ ((r >> sh) & (nc - 1))).expand(npad, nc, 8)
    return torch.gather(t, 1, src).contiguous().view(-1)


def _swizzled_image(wt_bf16):
    """[npad, kp] bf16 (W^T, K-major) -> the fused kernel's operand image: nfull blocks of [npad x 128 bytes] followed
    by the tail block of [npad x rbt bytes] (zero padded), each block swizzled over its own row span."""
    npad, kp = wt_bf16.shape
    nfull, rbt = _k_blocks(kp)
    parts = [_swizzle_block(wt_bf16[:, 64 * i: 64 * (i + 1)].contiguous(), 128) for i in range(nfull)]
    if rbt:
        tail = torch.zeros((npad, rbt // 2), dtype=torch.bfloat16, device=wt_bf16.device)
        tail[:, : kp - 64 * nfull] = wt_bf16[:, 64 * nfull:]
        parts.append(_swizzle_block(tail, rbt))
    return torch.cat(parts)


class FusedStack:
    """Operands of ssd3d_sa_mlp_fused for one SA scale: the split, pre-swizzled weight images of its conv layers
    packed as { hi | lo } per layer, and the folded { scale | shift } per layer (zero beyond the true width)."""

    def __init__(self, convs, cin):
        dev = convs[0].w.device
        self.nout = [f.cout for f in convs]
        self.cin = cin
        self.convs = list(convs)            # the folded layers the blobs were built from (introspection / CPU dry runs)
        # The LAST layer is stored with non-negative scales: (x.w) * s + t == (x.(w * sgn s)) * |s| + t, exactly (a sign
        # flip is exact in bf16).  fma(acc, |s|, t) is then monotone in acc, so the kernel may max-pool the raw
        # accumulators and apply scale / shift / ReLU to the pooled values only (ssd3d.h: last_scale_nonneg).
        self.last_scale_nonneg = True
        wparts, sparts = [], []
        kp = round16(cin)
        for li, f in enumerate(convs):
            npad = round16(f.cout)
            assert f.kp == kp, (f.kp, kp)
            b_hi, b_lo, scale = f.b_hi, f.b_lo, f.scale
            if li == len(convs) - 1:
                sgn = torch.where(scale < 0, -torch.ones_like(scale), torch.ones_like(scale))
                b_hi = (b_hi.float() * sgn.unsqueeze(1)).to(torch.bfloat16)
                b_lo = (b_lo.float() * sgn.unsqueeze(1)).to(torch.bfloat16)
                scale = scale.abs()
            hi = torch.zeros((npad, kp), dtype=torch.bfloat16, device=dev)
            lo = torch.zeros_like(hi)
            hi[: f.cout] = b_hi
            lo[: f.cout] = b_lo
            wparts += [_swizzled_image(hi), _swizzled_image(lo)]
            sspad = (npad + 31) // 32 * 32                 # the kernel reads scale/shift in 32-column chunks
            sc = torch.zeros(sspad, dtype=torch.float32, device=dev)
            sh = torch.zeros(sspad, dtype=torch.float32, device=dev)
            sc[: f.cout] = scale
            sh[: f.cout] = f.shift
            sparts += [sc, sh]
            kp = npad
        self.w_blob = torch.cat(wparts).contiguous()
        self.ss_blob = torch.cat(sparts).contiguous()


class PreparedParams:
    """Device-resident folded weights, looked up by TF scope name (lazy, cached)."""

    def __init__(self, params, device):
        self.raw = params
        self.device = torch.device(device)
        self._cache = {}

    def conv(self, scope, bn=True):
        key = (scope, bool(bn))
        if key not in self._cache:
            self._cache[key] = fold(self.raw, scope, bn, self.device)
        return self._cache[key]

    def fused_stack(self, scopes, bn, cin, limit=None):
        """FusedStack for a list of conv scopes (one SA scale), or None when the stack does not fit the fused kernel
        (limit = shared-memory bytes the policy allows; default FUSED_SMEM_LIMIT, pass 0 for 'whatever fits')."""
        limit = FUSED_SMEM_LIMIT if limit is None else (limit or 1 << 30)
        key = ("fused",) + tuple(scopes) + (bool(bn), cin, limit)
        if key not in self._cache:
            import ctypes
            from ._lib import lib
            convs = [self.conv(sc, bn) for sc in scopes]
            nout = (ctypes.c_int * len(convs))(*[f.cout for f in convs])
            need = lib().ssd3d_sa_fused_smem(cin - 3, len(convs), ctypes.cast(nout, ctypes.c_void_p)) if len(convs) <= 3 else 0
            # the fused kernel keeps every layer's weights in shared memory; stacks that do not fit (layer3/4 sized)
            # return None and take the layer-by-layer tensor-core path
            fits = 0 < need <= limit
            self._cache[key] = FusedStack(convs, cin) if fits else None
        return self._cache[key]

    def hoisted(self, scopes, bn, c):
        """First convs of the scales of one SA layer (scopes), hoisted: returns (FoldedConv for the per-point table
        z = (f . [Wf_1 | Wf_2 | ...]) * s + t over all scales, [Wx_i * s_i as (3, n1_i) per scale], [n1_i]).
        c = feature channels (the convs take c + 3 inputs: features first, then xyz - centre)."""
        key = ("hoisted",) + tuple(scopes) + (bool(bn), c)
        if key not in self._cache:
            convs = [self.conv(sc, bn) for sc in scopes]
            for f in convs:
                if f.cin != c + 3:
                    raise ValueError("hoisted: conv expects %d inputs, got c + 3 = %d" % (f.cin, c + 3))
            wf = torch.cat([f.w[:c] for f in convs], dim=1).contiguous()
            zconv = FoldedConv(wf, torch.cat([f.scale for f in convs]).contiguous(), torch.cat([f.shift for f in convs]).contiguous())
            wxs = [(f.w[c:c + 3].double() * f.scale.double().unsqueeze(0)).float().contiguous() for f in convs]
            self._cache[key] = (zconv, wxs, [f.cout for f in convs])
        return self._cache[key]

    # ---- training mode: BatchNorm state lives on the device and is updated in place by the forward -----------------
    def bn_state(self, scope):
        """{gamma, beta, moving_mean, moving_variance} of `scope` as device tensors; training-mode forwards update the
        moving statistics in place.  commit_bn() writes them back to the parameter dict."""
        key = ("bn_state", scope)
        if key not in self._cache:
            self._cache[key] = {k: torch.from_numpy(np.ascontiguousarray(self.raw[scope + "/bn/" + k], dtype=np.float32)).to(self.device)
                                for k in ("gamma", "beta", "moving_mean", "moving_variance")}
        return self._cache[key]

    def commit_bn(self):
        """Copy the moving statistics updated by training-mode forwards back into the raw parameter dict and drop every
        folded form derived from the old ones (inference after training folds the new statistics)."""
        touched = False
        for key in [k for k in self._cache if isinstance(k, tuple) and k[0] == "bn_state"]:
            st = self._cache[key]
            for k in ("moving_mean", "moving_variance"):
                self.raw[key[1] + "/bn/" + k] = st[k].detach().cpu().numpy()
            touched = True
        if touched:
            for key in [k for k in self._cache if not (isinstance(k, tuple) and k[0] == "bn_state")]:
                del self._cache[key]
        return self

    def prepare_all(self):
        for k in self.raw:
            if k.endswith("/weights"):
                scope = k[: -len("/weights")]
                self.conv(scope, (scope + "/bn/gamma") in self.raw)
        return self


def trained_names(names, prefixes=None):
    """The variables of `names` that training updates, as the reference's TRAIN.CONFIG.TRAIN_PARAM_PREFIX selects them
    (lib/core/trainer.py:42, trainer_utils.get_trainable_parameter: the scope filter of tf.get_collection): name v is
    trained iff re.match(prefix, v) for some prefix.  None or [] trains every name.  A prefix that matches no name is an
    error (a misspelt scope would otherwise freeze everything it meant to train).  Returns the trained names in the
    order of `names`."""
    import re
    names = list(names)
    if not prefixes:
        return names
    prefixes = [str(p) for p in prefixes]
    for p in prefixes:
        if not any(re.match(p, v) for v in names):
            raise ValueError("trainable prefix %r matches no variable (e.g. %s)" % (p, names[0] if names else "none"))
    return [v for v in names if any(re.match(p, v) for p in prefixes)]


class TrainableParams:
    """The parameters of a params dict as device tensors for training (layers with is_training=True run their
    differentiable path when given one of these): weights, biases, gamma and beta are leaf tensors with
    requires_grad=True, the moving statistics plain tensors that training forwards update in place.  Keys are the TF
    variable names.  Nothing folded is cached: every forward reads the live tensors, so an optimizer step is seen by the
    next forward.  to_params() returns the numpy dict (moving statistics included) for prepare() / SABackbone.

    trainable: the reference's TRAIN_PARAM_PREFIX (trained_names; None or [] trains everything).  A tensor it does not
    select is frozen: requires_grad=False, so autograd drops every layer below the lowest trained one and no gradient,
    clip, allreduce or optimizer slot covers it.  Frozen layers still run in training mode (batch statistics, moving
    statistics updated in place), as the reference's batch_norm_template does for every layer."""

    _STATS = ("/bn/moving_mean", "/bn/moving_variance")

    def __init__(self, params, device="cuda", trainable=None):
        self.device = torch.device(device)
        self.tensors = {}
        self.trainable = tuple(trainable) if trainable else ()
        trained = set(trained_names([k for k in params if not k.endswith(self._STATS)], self.trainable))
        for k, v in params.items():
            t = torch.from_numpy(np.array(v, dtype=np.float32, copy=True)).to(self.device)
            self.tensors[k] = t if k.endswith(self._STATS) else t.requires_grad_(k in trained)
        self.grad_flat = self.grad_offsets = None          # flat_grads()
        self.stats_flat = self.bn_offsets = None           # flat_stats()
        self._bn_record = None                             # start_bn_record() .. finish_bn_record()
        self._bn_sync = None                               # start_bn_sync() .. finish_bn_sync()
        self.param_flat = self.param_offsets = None        # flat_params()
        self.operand_cache = None                          # enable_operand_cache(): {scope: (forward fold, grad-x fold)}
        self.frozen_flat = None                            # enable_operand_cache(): the frozen weights, one buffer

    def named_parameters(self):
        """(TF name, tensor) of every trained tensor."""
        return [(k, t) for k, t in self.tensors.items() if t.requires_grad]

    def frozen_names(self):
        """Weights, biases, gamma and beta that training leaves alone (TrainableParams(trainable=...))."""
        return [k for k, t in self.tensors.items() if not (t.requires_grad or k.endswith(self._STATS))]

    def parameters(self):
        return [t for _, t in self.named_parameters()]

    def grads(self):
        """{TF name: gradient} of every trainable tensor (None where no gradient reached it)."""
        return {k: t.grad for k, t in self.named_parameters()}

    def to_params(self):
        return {k: t.detach().cpu().numpy().copy() for k, t in self.tensors.items()}

    def conv_train(self, scope, x, bn=True, bn_decay=None, relu=True, debug=None):
        """One conv (+ training BatchNorm when bn) (+ ReLU) of `scope`, differentiable (tf_ops.conv_train).  While a BN
        record is open (start_bn_record) the batch statistics go to the record instead of the moving statistics; while a
        BN sync is open (start_bn_sync) the BatchNorm is synchronised over the ranks of its handle (SyncBN)."""
        from . import tf_ops
        t = self.tensors
        g = lambda k: t.get(scope + k)
        b = g("/biases")
        if b is None:
            b = torch.zeros((t[scope + "/weights"].shape[1],), dtype=torch.float32, device=self.device)
        decay = 0.9 if bn_decay is None else float(bn_decay)
        moving, stats_out = (g("/bn/moving_mean"), g("/bn/moving_variance")), None
        if bn and self._bn_record is not None:
            stats_out, moving = self._record_slot(scope, decay), (None, None)
        extra = {} if self.operand_cache is None else {"operands": self.operand_cache[scope]}
        if bn and self._bn_sync is not None:
            self._claim(self._bn_sync, "BN sync", scope, decay)
            extra["sync"] = self._bn_sync["handle"].slots(scope)
        return tf_ops.conv_train(x, t[scope + "/weights"], b, g("/bn/gamma"), g("/bn/beta"), moving[0], moving[1], bn=bn, relu=relu,
                                 decay=decay, debug=debug, stats_out=stats_out, **extra)

    # ---- the solver (solver.Adam): both capabilities are opt-in; unused, nothing above changes ------------------------
    def flat_params(self):
        """Move every trainable tensor into ONE flat float32 buffer (param_flat; param_offsets[name] = its first element,
        the offsets of flat_grads): the tensors stay autograd leaves and become views of it, so one kernel can update all
        of them.  Returns param_flat."""
        if self.param_flat is None:
            self.param_flat, self.param_offsets = self._flatten(self.named_parameters())
        return self.param_flat

    def _flatten(self, named):
        """Move the tensors of `named` into one new flat float32 buffer (they become views of it and stay autograd
        leaves) -> (buffer, {name: its first element})."""
        flat = torch.empty((sum(t.numel() for _, t in named),), dtype=torch.float32, device=self.device)
        offsets, off = {}, 0
        for k, t in named:
            view = flat[off:off + t.numel()].view(t.shape)
            view.copy_(t.detach())
            t.data = view
            offsets[k] = off
            off += t.numel()
        return flat, offsets

    def weight_scopes(self):
        """Scopes of the trained conv weights."""
        return [k[: -len("/weights")] for k, _ in self.named_parameters() if k.endswith("/weights")]

    def frozen_weight_scopes(self):
        return [k[: -len("/weights")] for k in self.frozen_names() if k.endswith("/weights")]

    def enable_operand_cache(self):
        """Keep the split tensor-core operands of every conv weight in a bf16 arena (operand_layout) and hand them to
        conv_train instead of rebuilding them in every forward and backward.  The cache holds what refresh_operands() last
        built: it is valid from then until the next write to a weight, so whatever writes weights calls refresh_operands()
        (solver.Adam.step does).  The biases are read live (shift is a view of them).  Frozen weights move into a second
        flat buffer (frozen_flat) with an arena of its own whose rows are built here once: refresh_operands() rebuilds
        only the trained weights' rows unless told that the frozen weights were written too (a load or a broadcast)."""
        if self.operand_cache is not None:
            return
        self.flat_params()
        frozen = self.frozen_weight_scopes()
        self.frozen_flat, frozen_offsets = self._flatten([(s + "/weights", self.tensors[s + "/weights"]) for s in frozen])
        self.operand_cache = {}
        self._operands = [self._operand_rows(self.weight_scopes(), self.param_flat, self.param_offsets),
                          self._operand_rows(frozen, self.frozen_flat, frozen_offsets)]
        self.operand_arena = None if self._operands[0] is None else self._operands[0][3]
        self.refresh_operands(frozen=True)

    def _operand_rows(self, scopes, flat, offsets):
        """Operand cache entries for the weights of `scopes`, which live in `flat` at `offsets` -> the arguments of
        tf_ops.weight_operands that rebuild them (flat, table, tiles, arena), or None without a scope."""
        if not scopes:
            return None
        shapes = [tuple(self.tensors[s + "/weights"].shape) for s in scopes]
        table, elems, tiles = operand_layout([(offsets[s + "/weights"], ci, co) for s, (ci, co) in zip(scopes, shapes)])
        arena = torch.zeros((elems,), dtype=torch.bfloat16, device=self.device)
        width = max(max(sh) for sh in shapes)
        ones = torch.ones((width,), dtype=torch.float32, device=self.device)
        zeros = torch.zeros((width,), dtype=torch.float32, device=self.device)
        for s, (ci, co), row in zip(scopes, shapes, table.tolist()):
            w = self.tensors[s + "/weights"].detach()
            b = self.tensors.get(s + "/biases")
            blk = lambda o, r, c: arena[o:o + r * c].view(r, c)
            fwd = FoldedConv.from_operands(w, ones[:co], zeros[:co] if b is None else b.detach(),
                                           blk(row[3], co, round16(ci)), blk(row[4], co, round16(ci)))
            bwd = FoldedConv.from_operands(w.t(), ones[:ci], zeros[:ci], blk(row[5], ci, round16(co)), blk(row[6], ci, round16(co)))
            self.operand_cache[s] = (fwd, bwd)
        return flat, torch.from_numpy(table).to(self.device), tiles, arena

    def refresh_operands(self, frozen=False):
        """Rebuild the operand cache of the trained weights from their current values (one launch), with frozen=True that
        of the frozen weights too (one more); nothing to do when the cache is not enabled."""
        if self.operand_cache is not None:
            from . import tf_ops
            for rows in self._operands[:2 if frozen else 1]:
                if rows is not None:
                    tf_ops.weight_operands(*rows)

    # ---- data-parallel training (dist.DataParallel): both capabilities are opt-in; unused, nothing above changes -----
    def flat_grads(self):
        """Make every trainable tensor's .grad a view of ONE flat float32 buffer (grad_flat; grad_offsets[name] = the
        view's first element, in named_parameters order), so autograd accumulates in place and zeroing is one fill.
        Returns grad_flat."""
        if self.grad_flat is None:
            named = self.named_parameters()
            self.grad_flat = torch.zeros((sum(t.numel() for _, t in named),), dtype=torch.float32, device=self.device)
            self.grad_offsets, off = {}, 0
            for k, t in named:
                self.grad_offsets[k] = off
                off += t.numel()
        self._attach_grads()
        return self.grad_flat

    def _attach_grads(self):
        for k, t in self.named_parameters():
            o = self.grad_offsets[k]
            t.grad = self.grad_flat[o:o + t.numel()].view(t.shape)

    def zero_flat_grads(self):
        """grad_flat[:] = 0 (one kernel) and every .grad back on its view (an optimizer may have set it to None)."""
        from . import tf_ops
        tf_ops.fill_zero(self.grad_flat)
        self._attach_grads()

    def bn_scopes(self):
        return [k[: -len(self._STATS[0])] for k in self.tensors if k.endswith(self._STATS[0])]

    def flat_stats(self):
        """Move the moving statistics into ONE flat float32 buffer (stats_flat): scope s holds [moving_mean | moving_variance]
        at bn_offsets[s] = (offset, channels), in bn_scopes() order; the tensors become views of it.  Returns stats_flat."""
        if self.stats_flat is None:
            scopes = self.bn_scopes()
            sizes = [self.tensors[s + self._STATS[0]].numel() for s in scopes]
            flat = torch.empty((2 * sum(sizes),), dtype=torch.float32, device=self.device)
            self.bn_offsets, off = {}, 0
            for s, c in zip(scopes, sizes):
                self.bn_offsets[s] = (off, c)
                for i, suffix in enumerate(self._STATS):
                    v = flat[off + i * c: off + (i + 1) * c]
                    v.copy_(self.tensors[s + suffix])
                    self.tensors[s + suffix] = v
                off += 2 * c
            self.stats_flat = flat
        return self.stats_flat

    def start_bn_record(self, record):
        """Open a BN record: until finish_bn_record(), every training BatchNorm leaves the moving statistics alone and
        writes its batch mean and variance into `record` (float32 CUDA [>= stats_flat.numel()]) at its scope's
        bn_offsets, i.e. record mirrors stats_flat.  The record's views are kept for the backward of that forward."""
        self.flat_stats()
        if not isinstance(record, torch.Tensor) or record.dtype != torch.float32 or record.dim() != 1 or \
                record.numel() < self.stats_flat.numel() or record.device != self.stats_flat.device:
            raise ValueError("start_bn_record: record must be a float32 vector of >= %d elements on %s"
                             % (self.stats_flat.numel(), self.stats_flat.device))
        if self._bn_record is not None or self._bn_sync is not None:
            raise ValueError("start_bn_record: a BN record or BN sync is already open")
        self._bn_record = {"buf": record, "seen": set(), "decay": None}

    def _claim(self, rec, what, scope, decay):
        """The once-per-scope, one-decay bookkeeping of an open BN record or BN sync."""
        if scope not in self.bn_offsets:
            raise ValueError("%s: %s has no moving statistics" % (what, scope))
        if scope in rec["seen"]:
            raise ValueError("%s: %s recorded twice in one step" % (what, scope))
        if rec["decay"] is not None and decay != rec["decay"]:
            raise ValueError("%s: %s uses decay %g, the step uses %g" % (what, scope, decay, rec["decay"]))
        rec["seen"].add(scope)
        rec["decay"] = decay

    def _record_slot(self, scope, decay):
        rec = self._bn_record
        self._claim(rec, "BN record", scope, decay)
        off, c = self.bn_offsets[scope]
        return rec["buf"][off:off + c], rec["buf"][off + c:off + 2 * c]

    def finish_bn_record(self, check=True):
        """Close the BN record and return its decay.  check: every BN scope must have recorded exactly once."""
        rec, self._bn_record = self._bn_record, None
        if rec is None:
            raise ValueError("finish_bn_record: no BN record is open")
        return self._finish(rec, "BN record", check)

    def _finish(self, rec, what, check):
        missing = [s for s in self.bn_offsets if s not in rec["seen"]]
        if check and missing:
            raise ValueError("%s: %d scope(s) did not record, e.g. %s" % (what, len(missing), missing[0]))
        return rec["decay"]

    def start_bn_sync(self, handle):
        """Open a BN sync: until finish_bn_sync(), every training BatchNorm runs SyncBN over the ranks of `handle`
        (dist.BnSync: handle.slots(scope) -> the scope's (forward, backward) tf_ops.BnSyncSlot) and updates the moving
        statistics in place with the statistics of every rank's rows.  Each scope exactly once, with one decay."""
        self.flat_stats()
        if not callable(getattr(handle, "slots", None)):
            raise ValueError("start_bn_sync: handle must be a dist.BnSync")
        if self._bn_sync is not None or self._bn_record is not None:
            raise ValueError("start_bn_sync: a BN sync or BN record is already open")
        self._bn_sync = {"handle": handle, "seen": set(), "decay": None}

    def finish_bn_sync(self, check=True):
        """Close the BN sync and return its decay.  check: every BN scope must have been synchronised exactly once."""
        rec, self._bn_sync = self._bn_sync, None
        if rec is None:
            raise ValueError("finish_bn_sync: no BN sync is open")
        return self._finish(rec, "BN sync", check)


def prepare(params, device="cuda"):
    """Folded inference form of a params dict; a TrainableParams is folded from its current values."""
    if isinstance(params, TrainableParams):
        return PreparedParams(params.to_params(), device)
    return params if isinstance(params, PreparedParams) else PreparedParams(params, device)
