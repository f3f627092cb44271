"""The reference's solver on the GPU (DESIGN.md section 3.11): the SOLVER block of configs/kitti/3dssd/3dssd.yaml as
data, its two step-driven schedules, Adam over the flat parameter buffer (csrc/solver.cu), the training loop body of
lib/core/trainer.py:177-207 and checkpoints keyed by the reference's TF variable names.

    tp = params.TrainableParams(init, device)
    tr = solver.Trainer(config.ARCH_3DSSD, tp, solver.Solver())      # dp=dist.DataParallel(tp, arena) for several GPUs
    for xyz, feat, gt_boxes, gt_labels in batches:
        losses = tr.step(xyz, feat, gt_boxes, gt_labels)             # nothing in a step synchronises the host
    tr.save("model-00000807.npz")                                    # Trainer.load resumes from it bit for bit
"""
import bisect
import struct
from dataclasses import dataclass
from typing import Tuple

import numpy as np
import torch

SLOT_M, SLOT_V = "/Adam", "/Adam_1"           # tf.train.AdamOptimizer's slot variables of <var>
SCALARS = ("beta1_power", "beta2_power", "global_step")


@dataclass(frozen=True)
class Solver:
    """SOLVER of 3dssd.yaml:18-33 (TYPE 'Adam').  There is no weight decay: no layer of the 3DSSD model passes
    weight_decay to tf_util.conv2d / conv1d, so the reference's loss has no L2 term."""
    base_lr: float = 0.002
    steps: Tuple[int, ...] = (64560,)
    gamma: float = 0.1
    bn_init_decay: float = 0.5
    bn_decay_decay_rate: float = 0.5
    bn_decay_clip: float = 0.99
    beta1: float = 0.9
    beta2: float = 0.999
    epsilon: float = 1e-8
    clip_norm: float = 5.0
    max_iterations: int = 80700
    checkpoint_interval: int = 807

    def __post_init__(self):
        steps = tuple(int(s) for s in self.steps)
        if len(steps) > 8 or any(b <= a for a, b in zip(steps, steps[1:])):
            raise ValueError("Solver: steps must be at most 8 increasing boundaries, got %r" % (steps,))
        object.__setattr__(self, "steps", steps)

    def _piecewise(self, step, base, rate):
        """tf.train.piecewise_constant(step, steps, values) with the reference's values: Python doubles base * rate **
        (i + 1), cast to float32 by TF.  values[i] holds while steps[i-1] < step <= steps[i]."""
        values = [np.float32(base)] + [np.float32(base * rate ** (i + 1)) for i in range(len(self.steps))]
        return values[bisect.bisect_left(self.steps, int(step))]

    def lr_values(self):
        return [float(np.float32(self.base_lr))] + [float(np.float32(self.base_lr * self.gamma ** (i + 1)))
                                                    for i in range(len(self.steps))]

    def learning_rate(self, step):
        """float32 learning rate of the update that reads global_step == step (trainer_utils.py:7-13).  The reference's
        tf.maximum(learning_rate, 1e-5) is assigned to a misspelt name (`learing_rate`, trainer_utils.py:12) and never
        takes effect, so no floor is applied here either."""
        return self._piecewise(step, self.base_lr, self.gamma)

    def bn_decay(self, step):
        """float32 BatchNorm decay of the forward at global_step == step (trainer_utils.py:15-21):
        min(bn_decay_clip, 1 - momentum) in float32, momentum on the learning rate's boundaries."""
        momentum = self._piecewise(step, self.bn_init_decay, self.bn_decay_decay_rate)
        return min(np.float32(self.bn_decay_clip), np.float32(np.float32(1.0) - momentum))


def pack_state(global_step, beta1_power, beta2_power, lr_used=0.0):
    """The 32-byte device state block of ssd3d_adam_step as int32 [8]."""
    return np.frombuffer(struct.pack("<qfffIII", int(global_step), float(beta1_power), float(beta2_power), float(lr_used), 0, 0, 0),
                         np.int32).copy()


def unpack_state(words):
    """int32 [8] -> (global_step, beta1_power, beta2_power, lr_used), the floats as numpy float32."""
    step, b1, b2, lr = struct.unpack("<qfff", np.asarray(words, np.int32).tobytes()[:20])
    return step, np.float32(b1), np.float32(b2), np.float32(lr)


class Adam:
    """tf.train.AdamOptimizer over tp's flat parameter buffer: owns the moments m and v and the device state block.
    step() is two launches whatever the layer count: the update, then the rebuild of the operand cache it invalidated."""

    def __init__(self, tp, solver):
        self.tp, self.solver = tp, solver
        self.param, self.grad = tp.flat_params(), tp.flat_grads()
        self.m, self.v = torch.zeros_like(self.param), torch.zeros_like(self.param)
        self.state = torch.from_numpy(pack_state(0, np.float32(solver.beta1), np.float32(solver.beta2))).to(tp.device)
        tp.enable_operand_cache()                                  # the first forward precedes any update

    def step(self):
        from . import tf_ops
        s = self.solver
        tf_ops.adam_step(self.param, self.grad, self.m, self.v, self.state, s.steps, s.lr_values(), s.beta1, s.beta2, s.epsilon)
        self.tp.refresh_operands()

    def state_dict(self):
        """{m, v [n] float32, global_step, beta1_power, beta2_power, lr_used} as numpy.  Synchronises."""
        step, b1, b2, lr = unpack_state(self.state.cpu().numpy())
        return {"m": self.m.cpu().numpy(), "v": self.v.cpu().numpy(), "global_step": step, "beta1_power": b1, "beta2_power": b2,
                "lr_used": lr}

    def load_state_dict(self, sd):
        with torch.no_grad():
            for name, buf in (("m", self.m), ("v", self.v)):
                a = np.ascontiguousarray(sd[name], np.float32)
                if a.shape != tuple(buf.shape):
                    raise ValueError("Adam.load_state_dict: %s has shape %s, expected %s" % (name, a.shape, tuple(buf.shape)))
                buf.copy_(torch.from_numpy(a))
            self.state.copy_(torch.from_numpy(pack_state(sd["global_step"], sd["beta1_power"], sd["beta2_power"],
                                                         sd.get("lr_used", 0.0))))


def _variables(named, tensors, offsets, adam_state):
    """The variables of a checkpoint by TF name: every tensor of the model (numpy dict), the slots <var>/Adam and
    <var>/Adam_1 cut from the flat moments at the parameters' offsets, and beta1_power, beta2_power, global_step."""
    out ={k: np.asarray(v, np.float32) for k, v in tensors.items()}
    for k, shape in named:
        o, n = offsets[k], int(np.prod(shape))
        out[k + SLOT_M] = adam_state["m"][o:o + n].reshape(shape)
        out[k + SLOT_V] = adam_state["v"][o:o + n].reshape(shape)
    out["beta1_power"] = np.float32(adam_state["beta1_power"])
    out["beta2_power"] = np.float32(adam_state["beta2_power"])
    out["global_step"] = np.int64(adam_state["global_step"])
    return out


def _from_variables(named, offsets, n, variables):
    """Inverse of _variables for the optimizer's part: the Adam state dict of a checkpoint's variables."""
    m, v = np.zeros((n,), np.float32), np.zeros((n,), np.float32)
    for k, shape in named:
        for slot, flat in ((SLOT_M, m), (SLOT_V, v)):
            if k + slot not in variables:
                raise ValueError("checkpoint has no %s" % (k + slot))
            a = np.asarray(variables[k + slot], np.float32)
            if a.shape != tuple(shape):
                raise ValueError("%s has shape %s, expected %s" % (k + slot, a.shape, tuple(shape)))
            flat[offsets[k]:offsets[k] + a.size] = a.reshape(-1)
    for k in SCALARS:
        if k not in variables:
            raise ValueError("checkpoint has no %s" % k)
    return {"m": m, "v": v, "global_step": int(variables["global_step"]), "beta1_power": np.float32(variables["beta1_power"]),
            "beta2_power": np.float32(variables["beta2_power"])}


class Trainer:
    """The loop body of the reference's trainer (trainer.py:177-207) for one rank: forward at the scheduled BatchNorm
    decay, targets, the six losses, backward, the clip / allreduce / BN update of dist.DataParallel, and the Adam step.
    dp: a dist.DataParallel over tp for several GPUs; None trains on one GPU through the same exchange at world size 1
    (its clip is the pinned one and its BN update equals the in-place one bit for bit)."""

    def __init__(self, arch, tp, solver, dp=None):
        from . import dist
        self.arch, self.tp, self.solver = arch, tp, solver
        self.adam = Adam(tp, solver)
        if dp is None:
            self._sym = torch.zeros((dist.DataParallel.symmetric_bytes(tp, 1),), dtype=torch.uint8, device=tp.device)
            dp = dist.DataParallel(tp, peers=[self._sym.data_ptr()], world=1, rank=0, clip_norm=solver.clip_norm)
        elif dp.tp is not tp:
            raise ValueError("Trainer: dp must be the DataParallel of the same TrainableParams")
        self.dp = dp
        tp.refresh_operands()                # a DataParallel's constructor may have broadcast rank 0's weights
        self.global_step = 0                 # host mirror of the device's global_step: schedules need no device read

    def step(self, xyz, feat, gt_boxes, gt_labels):
        """One training step on this rank's scenes -> {loss name: 0-d tensor}, averaged over the ranks."""
        from . import backbone, loss
        decay = float(self.solver.bn_decay(self.global_step))
        self.dp.zero_grad()
        with self.dp.recording():
            o = backbone.train_forward(self.arch, self.tp, xyz, feat, bn_decay=decay)
        tg = loss.assign_targets(o.base_xyz, o.vote_base, gt_boxes, gt_labels)
        losses = loss.detection_loss(o.base_xyz, *o.head, o.vote_offsets[-1], tg)
        losses["total"].backward()
        mean = self.dp.exchange(losses)
        self.adam.step()
        self.global_step += 1
        return mean

    # ---- checkpoints: .npz keyed by the reference's TF variable names ------------------------------------------------
    def _named(self):
        return [(k, tuple(t.shape)) for k, t in self.tp.named_parameters()]

    def variables(self):
        """Everything tf.train.Saver would write: <scope>/weights, /biases, /bn/{gamma, beta, moving_mean,
        moving_variance}, the slots <var>/Adam and <var>/Adam_1, beta1_power, beta2_power, global_step.  Synchronises."""
        return _variables(self._named(), self.tp.to_params(), self.tp.param_offsets, self.adam.state_dict())

    def save(self, path):
        """Write variables() to `path` (.npz).  kitti_io.params_from_tf_variables reads the file as it is (it drops the
        slots and counters), so a checkpoint serves prepare() / SABackbone / tools/eval_kitti.py directly."""
        with open(path, "wb") as f:
            np.savez(f, **self.variables())

    def _assign(self, variables, names):
        with torch.no_grad():
            for k in names:
                a = np.asarray(variables[k], np.float32)
                t = self.tp.tensors[k]
                if a.ndim > 2 and k.endswith("/weights"):          # TF stores [1, 1, cin, cout] / [1, cin, cout] kernels
                    a = a.reshape(a.shape[-2:])
                if a.shape != tuple(t.shape):
                    raise ValueError("%s has shape %s, expected %s" % (k, a.shape, tuple(t.shape)))
                t.copy_(torch.from_numpy(np.ascontiguousarray(a)))
        self.tp.refresh_operands()

    def load(self, path):
        """Resume: restore every variable of a file written by save(), the optimizer's state included."""
        with np.load(path) as z:
            variables = {k: z[k] for k in z.files}
        missing = [k for k in self.tp.tensors if k not in variables]
        if missing:
            raise ValueError("checkpoint lacks %d variable(s), e.g. %s" % (len(missing), missing[0]))
        sd = _from_variables(self._named(), self.tp.param_offsets, self.adam.param.numel(), variables)
        self._assign(variables, list(self.tp.tensors))
        if sd["global_step"] > 0:                                  # what the last launch before the save reported
            sd["lr_used"] = self.solver.learning_rate(sd["global_step"] - 1)
        self.adam.load_state_dict(sd)
        self.global_step = sd["global_step"]

    def warm_start(self, path):
        """Initialise from a pre-trained file as trainer.py:161-174 does: copy the variables whose names this model has;
        global_step and the optimizer's slots and powers are left alone, names the model lacks are ignored.  Returns the
        names copied."""
        with np.load(path) as z:
            variables = {(k[:-2] if k.endswith(":0") else k): z[k] for k in z.files}
        names = [k for k in self.tp.tensors if k in variables]
        self._assign(variables, names)
        return names
