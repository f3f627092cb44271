"""numpy restatement of the solver (3dssd_b200/csrc/solver.cu, 3dssd_b200/solver.py, DESIGN.md section 3.11).

The reference only CALLS TensorFlow here (tf.train.AdamOptimizer, tf.train.piecewise_constant: lib/core/trainer.py:74-75,
lib/core/trainer_utils.py:7-21), so there is no reference source to compile: the recipe below, every float32 operation
rounded once, is the contract the kernels reproduce bit for bit.
  lr      = values[number of boundaries < global_step]                               (read before the increment)
  alpha   = rn(rn(lr * rn(sqrt(rn(1 - beta2_power)))) / rn(1 - beta1_power))
  m'      = rn(m + rn(rn(g - m) * rn(1 - beta1)))
  v'      = rn(v + rn(rn(rn(g * g) - v) * rn(1 - beta2)))
  p'      = rn(p - rn(rn(m' * alpha) / rn(rn(sqrt(v')) + epsilon)))
  then      beta1_power = rn(beta1_power * beta1), beta2_power likewise, global_step += 1
  operand   hi = bf16_rne(w), lo = bf16_rne(w - float(hi)), of W^T [cout, round16(cin)] and of W [cin, round16(cout)]
"""
import numpy as np

F = np.float32


def piecewise_constant(step, boundaries, values):
    """tf.train.piecewise_constant: values[0] for step <= boundaries[0], values[i] for boundaries[i-1] < step <=
    boundaries[i], values[-1] beyond the last boundary."""
    assert len(values) == len(boundaries) + 1
    k = 0
    for b in boundaries:
        if step > b:
            k += 1
    return values[k]


def lr_values(base_lr=0.002, steps=(64560,), gamma=0.1):
    """trainer_utils.py:9: Python doubles, cast to float32 when TF makes them constants."""
    return [F(base_lr)] + [F(base_lr * gamma ** (i + 1)) for i in range(len(steps))]


def learning_rate(step, base_lr=0.002, steps=(64560,), gamma=0.1):
    return piecewise_constant(step, steps, lr_values(base_lr, steps, gamma))


def bn_decay(step, init=0.5, rate=0.5, clip=0.99, steps=(64560,)):
    """trainer_utils.py:15-21: minimum(clip, 1 - momentum) in float32."""
    momentum = piecewise_constant(step, steps, [F(init)] + [F(init * rate ** (i + 1)) for i in range(len(steps))])
    return np.minimum(F(clip), F(F(1.0) - momentum))


def new_state(beta1=0.9, beta2=0.999):
    return {"global_step": 0, "beta1_power": F(beta1), "beta2_power": F(beta2), "lr_used": F(0.0)}


def adam_step(p, g, m, v, state, boundaries=(), values=(0.001,), beta1=0.9, beta2=0.999, epsilon=1e-8):
    """One step in float32, every intermediate rounded -> (p', m', v', state')."""
    p, g, m, v = (np.asarray(a, F) for a in (p, g, m, v))
    b1, b2, eps = F(beta1), F(beta2), F(epsilon)
    lr = F(piecewise_constant(state["global_step"], boundaries, [F(x) for x in values]))
    with np.errstate(all="ignore"):
        alpha = F(F(lr * F(np.sqrt(F(F(1.0) - state["beta2_power"])))) / F(F(1.0) - state["beta1_power"]))
        m2 = (m + ((g - m).astype(F) * F(F(1.0) - b1)).astype(F)).astype(F)
        v2 = (v + (((g * g).astype(F) - v).astype(F) * F(F(1.0) - b2)).astype(F)).astype(F)
        p2 = (p - ((m2 * alpha).astype(F) / (np.sqrt(v2).astype(F) + eps).astype(F)).astype(F)).astype(F)
    st = {"global_step": state["global_step"] + 1, "beta1_power": F(state["beta1_power"] * b1),
          "beta2_power": F(state["beta2_power"] * b2), "lr_used": lr}
    return p2, m2, v2, st


def adam_step_f64(p, g, m, v, t, lr, beta1=0.9, beta2=0.999, epsilon=1e-8):
    """The same update rule (epsilon outside the bias correction) in float64 with exact powers; t = 1 for the first step."""
    p, g, m, v = (np.asarray(a, np.float64) for a in (p, g, m, v))
    alpha = lr * np.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)
    m2 = m + (g - m) * (1.0 - beta1)
    v2 = v + (g * g - v) * (1.0 - beta2)
    return p - m2 * alpha / (np.sqrt(v2) + epsilon), m2, v2


def bf16_rne(x):
    """float32 -> the float32 value of its bfloat16 rounding (round to nearest, ties to even); finite inputs."""
    u = np.asarray(x, F).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(F)


def bf16_bits(x):
    """The 16 stored bits of values that are exactly representable in bfloat16."""
    return (np.asarray(x, F).view(np.uint32) >> 16).astype(np.uint16)


def split_operand(w):
    """(hi, lo) uint16 bit patterns [cout, round16(cin)] of the K-major split of W^T for W [cin, cout], zero padded:
    what params.FoldedConv(w, ...) holds in b_hi / b_lo."""
    w = np.asarray(w, F)
    cin, cout = w.shape
    wt = np.zeros((cout, (cin + 15) // 16 * 16), F)
    wt[:, :cin] = w.T
    hi = bf16_rne(wt)
    lo = bf16_rne((wt - hi).astype(F))
    return bf16_bits(hi), bf16_bits(lo)
