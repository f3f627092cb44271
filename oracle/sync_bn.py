"""numpy restatement of SyncBN (3dssd_b200/csrc/bn.cu, ssd3d_bn_train_sync / ssd3d_bn_train_grad_sync; DESIGN.md
section 3.18) and a float64 restatement of the reference's sync_batch_norm (lib/utils/sync_bn.py) with num_dev = G.

Forward, pinned so that every rank holds the same bits:
  rank r: (rows_r, sum x_r, sum x_r^2) per channel in double, in the order of bn_partial_kernel and its fold
          (thread (rb, ty) adds rows rb*8 + ty + k*nrb*8 in k order, then ty = 0..7, then rb = 0..nrb-1)
  N, S1, S2 = the triples added in rank order 0..G-1 in double (rank 0's triple first)
  mean = S1 / N, var = max(S2 / N - mean^2, 0) in double, then bn.cu's float32 finalize (finalize below)
Backward: coef = (gamma r, sum_all g / N, sum_all g x^ / N, r) with r = 1 / sqrt(var + eps) in double; grad_x =
gamma r (g - sum_all g / N - x^ sum_all g x^ / N) per element; grad_gamma / grad_beta are the rank's own sums.
Moving statistics: bn.cu's in-place update, once per step, with the global (mean, var).
"""
from fractions import Fraction

import numpy as np

BN_TY, BN_MAX_RB = 8, 256


def nrb_of(rows):
    """Row blocks of bn.cu's partial kernel: >= 64 rows per thread before another block pays, 1..256."""
    return int(min(max(-(-int(rows) // (BN_TY * 64)), 1), BN_MAX_RB))


def _ordered_sums(vals):
    """vals [rows, k, c] float64 -> [k, c]: summed in bn_partial_kernel's order, then folded over the row blocks."""
    rows = vals.shape[0]
    nrb = nrb_of(rows)
    span = nrb * BN_TY
    steps = -(-rows // span)
    pad = np.zeros((steps * span,) + vals.shape[1:], dtype=np.float64)      # + 0.0 leaves every sum unchanged
    pad[:rows] = vals
    pad = pad.reshape((steps, nrb, BN_TY) + vals.shape[1:])
    acc = np.zeros(pad.shape[1:], dtype=np.float64)
    for k in range(steps):
        acc = acc + pad[k]
    blk = acc[:, 0]
    for i in range(1, BN_TY):
        blk = blk + acc[:, i]
    out = np.zeros(vals.shape[1:], dtype=np.float64)
    for rb in range(nrb):
        out = out + blk[rb]
    return out


def local_triple(x):
    """(rows, sum x, sum x^2) of one rank's rows x [rows, c] float32, each [c] float64, in the kernel's order."""
    x = np.asarray(x, dtype=np.float32)
    v = x.astype(np.float64)
    s = _ordered_sums(np.stack([v, v * v], axis=1))                      # v * v is exact in double
    return np.full(x.shape[1], float(x.shape[0])), s[0], s[1]


def rank_order_sum(triples):
    """The exchange: triples added in rank order, rank 0's first."""
    n, a, b = (np.array(t, dtype=np.float64, copy=True) for t in triples[0])
    for t in triples[1:]:
        n, a, b = n + t[0], a + t[1], b + t[2]
    return n, a, b


def rsqrt_rn(a):
    """float32 1/sqrt(a) correctly rounded (__frsqrt_rn), a float32 > 0."""
    a = np.asarray(a, dtype=np.float32)
    y = (1.0 / np.sqrt(a.astype(np.float64))).astype(np.float32)
    out = y.copy()
    for i in np.ndindex(a.shape):
        ai, yi = Fraction(float(a[i])), y[i]
        lo, hi = np.nextafter(yi, np.float32(0)), np.nextafter(yi, np.float32(np.inf))
        m_lo = (Fraction(float(lo)) + Fraction(float(yi))) / 2
        m_hi = (Fraction(float(yi)) + Fraction(float(hi))) / 2
        if m_hi * m_hi * ai < 1:
            out[i] = hi
        elif m_lo * m_lo * ai > 1:
            out[i] = lo
    return out


def finalize(n, s1, s2, gamma, beta, eps=1e-3):
    """bn.cu's finalize of sums over n rows -> (scale, shift, mean, var), float32 [c]."""
    mean_d = s1 / n
    var_d = np.maximum(s2 / n - mean_d * mean_d, 0.0)
    mean, var = mean_d.astype(np.float32), var_d.astype(np.float32)
    inv = np.asarray(gamma, np.float32) * rsqrt_rn(var + np.float32(eps))
    shift = np.asarray(beta, np.float32) - mean * inv
    return inv.astype(np.float32), shift.astype(np.float32), mean, var


def moving_update(moving, value, decay):
    """bn.cu's assign_moving_average: v -= (v - value) * (1 - decay), float32."""
    om = np.float32(1.0) - np.float32(decay)
    v = np.asarray(moving, dtype=np.float32)
    return (v - (v - np.asarray(value, np.float32)) * om).astype(np.float32)


def apply(x, scale, shift, relu=True):
    """The apply pass fma(x, scale, shift), then ReLU: the exact product plus shift rounded to double, then to float32
    (within one float32 rounding of fmaf; used with tolerances only)."""
    y = (np.asarray(x, np.float32).astype(np.float64) * scale.astype(np.float64) + shift.astype(np.float64)).astype(np.float32)
    return np.maximum(y, np.float32(0)) if relu else y


def bn_train_single(x, gamma, beta, eps=1e-3):
    """One rank's ssd3d_bn_train: the kernel's own fold and finalize over its rows alone."""
    n, a, b = local_triple(x)
    return finalize(n, a, b, gamma, beta, eps)


def forward(shards, gamma, beta, eps=1e-3):
    """SyncBN over the ranks' row blocks `shards` ([rows_r, c] float32 each) -> (scale, shift, mean, var) of every rank."""
    return finalize(*rank_order_sum([local_triple(x) for x in shards]), gamma, beta, eps)


def backward(shards, gouts, scale, shift, mean, var, gamma, relu=True, eps=1e-3):
    """SyncBN backward -> per rank (grad_x float32, grad_gamma float32, grad_beta float32).  The sums are float64 in
    natural order (the kernel's own order is pinned by the forward; here the tolerance of the caller applies)."""
    r = 1.0 / np.sqrt(np.asarray(var, np.float32).astype(np.float64) + np.float64(np.float32(eps)))
    mu = np.asarray(mean, np.float32).astype(np.float64)
    local, n_all, sg_all, sgx_all = [], 0.0, 0.0, 0.0
    for x, go in zip(shards, gouts):
        x = np.asarray(x, np.float32)
        g = np.asarray(go, np.float32).astype(np.float64)
        if relu:
            g = np.where(x.astype(np.float64) * scale.astype(np.float64) + shift.astype(np.float64) > 0, g, 0.0)
        xh = (x.astype(np.float64) - mu) * r
        local.append((g, xh, g.sum(0), (g * xh).sum(0)))
        n_all, sg_all, sgx_all = n_all + x.shape[0], sg_all + local[-1][2], sgx_all + local[-1][3]
    gr = np.asarray(gamma, np.float32).astype(np.float64) * r
    out = []
    for g, xh, sg, sgx in local:
        gx = gr * (g - sg_all / n_all - xh * (sgx_all / n_all))
        out.append((gx.astype(np.float32), sgx.astype(np.float32), sg.astype(np.float32)))
    return out


def reference_sync_batch_norm(shards, gamma, beta, moving_mean, moving_var, decay, eps=1e-3):
    """float64 restatement of the reference's sync_batch_norm (lib/utils/sync_bn.py) with num_dev = G = len(shards):
    mean = (sum_r mean_r) / G, mean_square = (sum_r mean(x_r^2)) / G, var = mean_square - mean^2, the outputs of
    tf.nn.batch_normalization per tower and device 0's moving update moving * decay + value * (1 - decay).  Returns
    (outputs per rank, mean, var, new moving_mean, new moving_var)."""
    g = len(shards)
    xs = [np.asarray(x, np.float64) for x in shards]
    mean = sum(x.mean(0) for x in xs) / g
    var = sum((x * x).mean(0) for x in xs) / g - mean * mean
    gm, bt = np.asarray(gamma, np.float64), np.asarray(beta, np.float64)
    outs = [(x - mean) / np.sqrt(var + eps) * gm + bt for x in xs]
    mm = np.asarray(moving_mean, np.float64) * decay + mean * (1 - decay)
    mv = np.asarray(moving_var, np.float64) * decay + var * (1 - decay)
    return outs, mean, var, mm, mv
