"""CPU tests of the host-side operand preparation of the grouped MLP (3dssd_b200/params.py): the pre-swizzled weight
images, the bf16 hi/lo split and its error budget, and the sign folding that lets the fused kernel pool before the affine.
They pin what the tensor-core kernels are fed; the kernels themselves are parity-tested on the GPU
(tests/test_ops_gpu.py).  The arithmetic restated: conv2d + bias + batch norm + ReLU + reduce_max of
/root/reference/lib/utils/tf_util.py:127-201,424-444 and /root/reference/lib/utils/layers_util.py:167-180."""
import importlib

import numpy as np
import pytest
import torch

P = importlib.import_module("3dssd_b200.params")


@pytest.mark.parametrize("rb", [128, 64, 32])
def test_swizzle_block_is_the_canonical_xor_of_address_bits(rb):
    """K-major wgmma / TMA shared-memory layouts SWIZZLE_128B / 64B / 32B XOR the 16-byte-chunk address bits [4, 4+B) with
    bits [7, 7+B) (B = 3 / 2 / 1): element (r, k) of a [rows, rb/2] bf16 block lives at byte a ^ (((a >> 7) & (2^B - 1)) << 4)
    with a = r * rb + 2k.  _swizzle_block is written in terms of chunks and row groups; this checks it address by address."""
    rows = 48
    cols = rb // 2
    blk = torch.arange(rows * cols, dtype=torch.float32).remainder(251).to(torch.bfloat16).reshape(rows, cols)
    img = P._swizzle_block(blk, rb).float().numpy()
    bits = {128: 3, 64: 2, 32: 1}[rb]
    r, k = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    a = r * rb + 2 * k
    a_sw = a ^ (((a >> 7) & ((1 << bits) - 1)) << 4)
    np.testing.assert_array_equal(img[a_sw // 2], blk.float().numpy())


def test_swizzled_image_block_structure():
    """kp = 80 -> one 64-column block (128-byte rows) + a 16-column tail block (32-byte rows): 40 KiB-per-256-rows, not 64."""
    assert P._k_blocks(80) == (1, 32) and P._k_blocks(64) == (1, 0) and P._k_blocks(96) == (1, 64) and P._k_blocks(112) == (1, 128)
    npad, kp = 32, 80
    wt = (torch.arange(npad * kp, dtype=torch.float32).remainder(199)).to(torch.bfloat16).reshape(npad, kp)
    img = P._swizzled_image(wt)
    assert img.numel() == npad * 64 + npad * 16
    np.testing.assert_array_equal(img[: npad * 64].float().numpy(), P._swizzle_block(wt[:, :64].contiguous(), 128).float().numpy())
    np.testing.assert_array_equal(img[npad * 64:].float().numpy(), P._swizzle_block(wt[:, 64:].contiguous(), 32).float().numpy())


def _split(x):
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def test_bf16_split_reconstructs_to_16_mantissa_bits():
    """x = hi + lo with two round-to-nearest bf16 terms leaves a relative error below 2^-16 (8 + 8 explicit mantissa bits
    and the sign of lo buys one more): the fp32-grade accuracy the three-MMA product rests on."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1 << 16, generator=g) * torch.exp(4 * torch.randn(1 << 16, generator=g))
    hi, lo = _split(x)
    rel = ((hi.double() + lo.double() - x.double()).abs() / x.double().abs()).max().item()
    assert rel < 2.0 ** -16
    f = P.FoldedConv(torch.randn(67, 64, generator=g), torch.ones(64), torch.zeros(64))
    assert f.kp == 80 and tuple(f.b_hi.shape) == (64, 80)
    assert float(f.b_hi[:, 67:].float().abs().max()) == 0.0 and float(f.b_lo[:, 67:].float().abs().max()) == 0.0
    w_rec = (f.b_hi.double() + f.b_lo.double())[:, :67].t()
    assert ((w_rec - f.w.double()).abs() / f.w.double().abs().clamp_min(1e-30)).max().item() < 2.0 ** -16


def test_three_term_split_product_meets_the_parity_budget_through_a_stack():
    """The kernels compute x.W as hi.hi + lo.hi + hi.lo in three bf16 MMAs with fp32 accumulation and re-split the
    activations between layers.  Emulated here in numpy/torch on the CPU for a layer-2-sized stack with KITTI-sized inputs:
    the relative error against float64 stays two orders of magnitude inside the 1e-3 budget of BASELINE.json, whereas one
    bf16 pass does not."""
    g = torch.Generator().manual_seed(1)
    rows, chans = 4096, [67, 64, 64, 128]
    feats = torch.relu(torch.randn(rows, 64, generator=g))
    dxyz = (torch.rand(rows, 3, generator=g) - 0.5) * 1.6            # xyz_j - c_i inside a 0.8 m ball
    x = torch.cat([feats, dxyz], 1)
    prm, rng = {}, np.random.default_rng(5)
    for j in range(3):
        P._conv_init(rng, prm, "s/conv0_%d" % j, chans[j], chans[j + 1], True)
    convs = [P.fold(prm, "s/conv0_%d" % j, True, "cpu") for j in range(3)]

    def run(mode):
        a = x.double() if mode == "f64" else x
        for f in convs:
            if mode == "f64":
                acc = a @ f.w.double()
                a = torch.relu(acc * f.scale.double() + f.shift.double())
                continue
            ah, al = _split(a)
            wh, wl = _split(f.w)
            if mode == "split3":
                acc = ah.float() @ wh.float() + al.float() @ wh.float() + ah.float() @ wl.float()
            else:
                acc = ah.float() @ wh.float()
            a = torch.relu(torch.addcmul(f.shift, acc, f.scale))
        return a.double()

    ref = run("f64")
    err3 = ((run("split3") - ref).abs().max() / ref.abs().max()).item()
    err1 = ((run("bf16") - ref).abs().max() / ref.abs().max()).item()
    assert err3 < 1e-5, err3
    assert err1 > 1e-3, err1                                         # why a single bf16 pass is not an option


def test_fused_stack_sign_fold_makes_pool_before_affine_exact():
    """FusedStack stores the last layer with non-negative scales: (x.w)*s + t == (x.(w*sgn s))*|s| + t, and with s >= 0
    the affine + ReLU is monotone, so max over the neighbours may be taken on the raw accumulators (layers_util.py:178
    reduce_max after the last conv).  Checked bit for bit in fp32, with negative gammas in the mix."""
    rng = np.random.default_rng(2)
    prm = {}
    P._conv_init(rng, prm, "s/conv0_0", 19, 32, True)
    P._conv_init(rng, prm, "s/conv0_1", 32, 48, True)
    prm["s/conv0_1/bn/gamma"][::3] *= -1.0                            # a third of the channels flip sign
    convs = [P.fold(prm, "s/conv0_%d" % j, True, "cpu") for j in range(2)]
    st = P.FusedStack(convs, 19)
    assert st.last_scale_nonneg and st.nout == [32, 48]
    last = convs[-1]
    assert bool((last.scale < 0).any())
    # the blob's scale / shift of the last layer: |s| and t
    off = 2 * 32                                                      # layer 0: 32 scales + 32 shifts (npad 32 -> chunk 32)
    sc, sh = st.ss_blob[off: off + 48], st.ss_blob[off + 64: off + 64 + 48]
    np.testing.assert_array_equal(sc.numpy(), last.scale.abs().numpy())
    np.testing.assert_array_equal(sh.numpy(), last.shift.numpy())
    groups, nsample = 64, 16
    a = torch.relu(torch.randn(groups, nsample, 32, generator=torch.Generator().manual_seed(3)))
    sgn = torch.where(last.scale < 0, -1.0, 1.0)
    acc = a @ last.w                                                   # [groups, nsample, 48] raw accumulators
    acc_folded = a @ (last.w * sgn)                                    # what the kernel accumulates
    np.testing.assert_array_equal(acc_folded.numpy(), (acc * sgn).numpy())   # a sign flip commutes with every rounding
    literal = torch.relu(torch.addcmul(last.shift, acc, last.scale)).amax(1)
    pooled_first = torch.relu(torch.addcmul(last.shift, acc_folded.amax(1), last.scale.abs()))
    np.testing.assert_array_equal(pooled_first.numpy(), literal.numpy())


def test_unit_list_rows_are_enough_for_the_max_pool():
    """A neighbour list with cnt hits holds cnt distinct rows and nsample - cnt copies of its first hit
    (tf_grouping_g.cu:245-248), so the max over the first 8*ceil(cnt/8) rows equals the max over all nsample rows --
    the identity behind the unit lists (DESIGN 3.4)."""
    rng = np.random.default_rng(4)
    n, m, nsample, c = 500, 200, 32, 24
    feats = rng.standard_normal((n, c)).astype(np.float32)
    cnt = rng.integers(0, nsample + 1, m)
    idx = np.zeros((m, nsample), np.int64)
    for q in range(m):
        if cnt[q]:
            hits = np.sort(rng.choice(n, cnt[q], replace=False))
            idx[q] = hits[0]                                           # back-fill with the first hit ...
            idx[q, : cnt[q]] = hits                                    # ... then the hits in index order
    act = np.maximum(feats[idx] @ rng.standard_normal((c, 16)).astype(np.float32), 0)    # any per-row function
    dense = act.max(1) * (cnt > 0)[:, None]
    compact = np.zeros_like(dense)                                     # the zero fill is the cnt == 0 mask
    for q in range(m):
        for j in range((cnt[q] + 7) // 8):                             # the units the ball query lists for group q
            compact[q] = np.maximum(compact[q], act[q, 8 * j: 8 * j + 8].max(0))
    np.testing.assert_array_equal(compact, dense)
