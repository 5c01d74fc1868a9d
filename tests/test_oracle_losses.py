"""The fp64 oracles of the L1 and SSIM losses (oracle/loss_oracle.py) and the host side of their CUDA entry points.
CPU only.

TensorFlow cannot be installed offline, so the SSIM oracle is pinned here by the window's definition, known answers
and an independent scipy restatement; its gradient by gradcheck.  A float32 emulation of TF's own formulation
(`tf_ssim_fp32`, the operation order of TF 2.2 `_ssim_helper`) measures what fp32 arithmetic costs TF on two input
families; those errors (EMUL_ERR) are the bars of the CUDA kernel in tests/test_gpu_ssim_l1.py."""
import numpy as np
import pytest
import torch
from scipy.signal import correlate2d

from oracle import loss_oracle as LO

C1, C2 = 0.01 ** 2, 0.03 ** 2

# Worst error of tf_ssim_fp32 against the fp64 oracle, per input family, at (2, 256, 256) (make_images seed 0):
# per-sample loss (absolute) and d_pred (relative Frobenius).  test_fp32_emulation_error_is_recorded re-measures them.
EMUL_ERR = {'noisy': {'loss': 2.894e-08, 'd_pred': 3.647e-06},
            'saturated': {'loss': 9.298e-07, 'd_pred': 7.772e-04}}


def make_images(family, B, H, W, seed=0):
    """float32 (gt, pred) [B, H, W, 3].  noisy: gt uniform on k/255, pred = gt + N(0, 0.05).  saturated: 48-pixel
    checkerboard squares flat at 254/255 (pred there = gt + N(0, 1e-3), where Cd is c2 plus a tiny variance and
    cancels worst), the other squares as noisy."""
    rng = np.random.default_rng(seed)
    gt = rng.integers(0, 256, size=(B, H, W, 3)) / 255.0
    if family == 'noisy':
        pred = gt + rng.normal(0, 0.05, size=gt.shape)
    elif family == 'saturated':
        yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing='ij')
        flat = np.broadcast_to(((yy // 48 + xx // 48) % 2 == 0)[None, :, :, None], gt.shape)
        gt = np.where(flat, 254 / 255, gt)
        pred = gt + np.where(flat, rng.normal(0, 1e-3, size=gt.shape), rng.normal(0, 0.05, size=gt.shape))
    else:
        raise ValueError(family)
    return gt.astype(np.float32), pred.astype(np.float32)


def tf_ssim_fp32(gt, pred, max_val=1.0, loss_scale=1.0):
    """numpy float32 emulation of tf.image.ssim + (1 - ssim) / 2 and of its gradient w.r.t. pred: the 121-tap window
    sums of the depthwise conv, TF 2.2 _ssim_helper's operation order, the adjoint in the same precision.
    Returns (loss [B], d(sum_b loss_b * loss_scale)/d(pred) [B, H, W, 3])."""
    f = np.float32
    x = np.ascontiguousarray(np.transpose(gt.astype(f), (0, 3, 1, 2)))
    y = np.ascontiguousarray(np.transpose(pred.astype(f), (0, 3, 1, 2)))
    G = LO.fspecial_gauss(dtype=torch.float32).numpy()
    n, c, h, w = x.shape
    hv, wv = h - 10, w - 10

    def red(t):
        out = np.zeros((n, c, hv, wv), f)
        for i in range(11):
            for j in range(11):
                out += G[i, j] * t[:, :, i:i + hv, j:j + wv]
        return out

    def red_t(t):
        out = np.zeros((n, c, h, w), f)
        for i in range(11):
            for j in range(11):
                out[:, :, i:i + hv, j:j + wv] += G[i, j] * t
        return out
    c1, c2 = f((f(0.01) * f(max_val)) ** 2), f((f(0.03) * f(max_val)) ** 2)
    m0, m1 = red(x), red(y)
    num0 = m0 * m1 * f(2)
    den0 = m0 * m0 + m1 * m1
    lum = (num0 + c1) / (den0 + c1)
    num1 = red(x * y) * f(2)
    den1 = red(x * x + y * y)
    cs = (num1 - num0 + c2) / (den1 - den0 + c2)
    ssim = (lum * cs).mean(axis=(2, 3), dtype=f).mean(axis=1, dtype=f)
    loss = (f(1) - ssim) / f(2)
    ld, cd = den0 + c1, den1 - den0 + c2
    wgt = f(-loss_scale / (2 * 3 * hv * wv))
    a = wgt * (f(2) * cs * (m0 - lum * m1) / ld + f(2) * lum * (cs * m1 - m0) / cd)
    bc = wgt * f(2) * lum / cd
    cc = -wgt * lum * cs / cd
    d = red_t(a) + x * red_t(bc) + f(2) * y * red_t(cc)
    return loss, np.transpose(d, (0, 2, 3, 1))


def ssim_ref64(gt, pred, loss_scale=1.0, device='cpu'):
    """fp64 oracle per-sample loss and d(sum_b loss_b * loss_scale)/d(pred) (autograd), as tensors on `device`."""
    g = torch.as_tensor(gt).to(device, torch.float64)
    p = torch.as_tensor(pred).to(device, torch.float64).requires_grad_(True)
    loss = LO.ssim_loss(g, p, keep_batch=True)
    (loss.sum() * loss_scale).backward()
    return loss.detach(), p.grad


def emul_errors(gt, pred):
    l32, d32 = tf_ssim_fp32(gt, pred)
    l64, d64 = (t.numpy() for t in ssim_ref64(gt, pred))
    return float(np.abs(l32 - l64).max()), float(np.linalg.norm(d32 - d64) / np.linalg.norm(d64))


# ---------------------------------------------------------------------------
# the window
# ---------------------------------------------------------------------------
def test_window_is_the_normalised_gaussian_and_separable():
    G = LO.fspecial_gauss().numpy()
    i = np.arange(-5, 6)
    e = np.exp(-(i[:, None] ** 2 + i[None, :] ** 2) / 4.5)
    np.testing.assert_allclose(G, e / e.sum(), rtol=0, atol=1e-15)
    assert abs(G.sum() - 1) < 1e-15 and G.shape == (11, 11)
    g1 = np.exp(-i ** 2 / 4.5)
    g1 /= g1.sum()
    np.testing.assert_allclose(G, np.outer(g1, g1), rtol=0, atol=1e-15)


# ---------------------------------------------------------------------------
# known answers
# ---------------------------------------------------------------------------
def test_ssim_of_an_image_with_itself_is_one():
    x = torch.rand(2, 17, 23, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    torch.testing.assert_close(LO.ssim(x, x), torch.ones(2, dtype=torch.float64), rtol=0, atol=1e-14)
    assert float(LO.ssim_loss(x, x).abs()) < 1e-14


@pytest.mark.parametrize('a,b', [(0.2, 0.7), (1.0, 0.0), (0.5, 0.5), (0.93, 0.95)])
def test_ssim_of_constant_images(a, b):
    gt = torch.full((1, 14, 12, 3), a, dtype=torch.float64)
    pred = torch.full((1, 14, 12, 3), b, dtype=torch.float64)
    lum, cs = LO.ssim_terms(gt, pred)
    want = (2 * a * b + C1) / (a * a + b * b + C1)
    assert lum.shape == (1, 3, 4, 2)
    torch.testing.assert_close(lum * cs, torch.full_like(lum, want), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(LO.ssim_loss(gt, pred, keep_batch=True), torch.tensor([(1 - want) / 2],
                                                                                    dtype=torch.float64))


def test_l1_known_answer_with_ties():
    gt = torch.tensor([[[[0.0, 0.5, 1.0], [0.25, 0.25, 0.25]],
                        [[1.0, 1.0, 0.0], [0.5, 0.0, 0.75]]]], dtype=torch.float64)
    pred = torch.tensor([[[[0.5, 0.5, 0.0], [0.25, 1.25, 0.0]],
                          [[1.0, 0.0, 0.0], [0.0, 0.5, 0.75]]]], dtype=torch.float64, requires_grad=True)
    # |d| = 0.5 0 1 | 0 1 0.25 | 0 1 0 | 0.5 0.5 0  -> sum 4.75 over 12 elements
    loss = LO.l1_loss(gt, pred, keep_batch=True)
    torch.testing.assert_close(loss, torch.tensor([4.75 / 12], dtype=torch.float64), rtol=0, atol=1e-15)
    loss.sum().backward()
    want = torch.tensor([[[[1, 0, -1], [0, 1, -1]], [[0, -1, 0], [-1, 1, 0]]]], dtype=torch.float64) / 12
    assert torch.equal(pred.grad, want)                        # ties give exactly 0


# ---------------------------------------------------------------------------
# independent restatement: scipy correlate2d per channel
# ---------------------------------------------------------------------------
def _scipy_ssim(gt, pred):
    i = np.arange(-5, 6)
    e = np.exp(-(i[:, None] ** 2 + i[None, :] ** 2) / 4.5)
    G = e / e.sum()
    out = []
    for b in range(gt.shape[0]):
        vals = []
        for c in range(3):
            x, y = gt[b, :, :, c], pred[b, :, :, c]
            f = lambda t: correlate2d(t, G, mode='valid')
            mx, my = f(x), f(y)
            vx, vy, cxy = f(x * x) - mx * mx, f(y * y) - my * my, f(x * y) - mx * my
            lum = (2 * mx * my + C1) / (mx * mx + my * my + C1)
            cs = (2 * cxy + C2) / (vx + vy + C2)
            vals.append((lum * cs).mean())
        out.append(np.mean(vals))
    return np.array(out)


@pytest.mark.parametrize('H,W', [(11, 11), (13, 12), (40, 23)])
def test_ssim_matches_an_independent_scipy_restatement(H, W):
    rng = np.random.default_rng(H * W)
    gt = rng.random((2, H, W, 3))
    pred = np.clip(gt + rng.normal(0, 0.1, gt.shape), 0, 1)
    got = LO.ssim(torch.from_numpy(gt), torch.from_numpy(pred)).numpy()
    np.testing.assert_allclose(got, _scipy_ssim(gt, pred), rtol=0, atol=1e-12)


# ---------------------------------------------------------------------------
# gradients and reductions
# ---------------------------------------------------------------------------
def test_oracle_gradients_pass_gradcheck_and_scalar_is_the_batch_mean():
    g = torch.Generator().manual_seed(3)
    gt = torch.rand(2, 13, 14, 3, dtype=torch.float64, generator=g)
    pred = (gt + 0.1 * torch.randn(2, 13, 14, 3, dtype=torch.float64, generator=g)).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda p: LO.ssim_loss(gt, p, keep_batch=True), (pred,))
    assert torch.autograd.gradcheck(lambda p: LO.l1_loss(gt, p, keep_batch=True), (pred,))   # no ties in random data
    for fn in (LO.ssim_loss, LO.l1_loss):
        torch.testing.assert_close(fn(gt, pred), fn(gt, pred, keep_batch=True).mean(), rtol=1e-15, atol=0)


def test_ssim_rejects_images_smaller_than_the_window():
    with pytest.raises(ValueError):
        LO.ssim_loss(torch.zeros(1, 10, 20, 3), torch.zeros(1, 10, 20, 3))
    with pytest.raises(ValueError):
        LO.ssim_loss(torch.zeros(1, 20, 10, 3), torch.zeros(1, 20, 10, 3))


# ---------------------------------------------------------------------------
# what fp32 costs TF's own formulation (sets the bars of the CUDA kernel)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('family', ['noisy', 'saturated'])
def test_fp32_emulation_error_is_recorded(family):
    gt, pred = make_images(family, 2, 256, 256)
    le, de = emul_errors(gt, pred)
    rec = EMUL_ERR[family]
    print('%s: tf fp32 emulation vs fp64: loss %.3e, d_pred rel Frobenius %.3e' % (family, le, de))
    assert rec['loss'] / 1.5 <= le <= rec['loss'] * 1.5, (le, rec)
    assert rec['d_pred'] / 1.5 <= de <= rec['d_pred'] * 1.5, (de, rec)
    # TF's cancellation in Cd: flat regions near 1 cost two orders of magnitude in d_pred
    assert EMUL_ERR['saturated']['d_pred'] > 100 * EMUL_ERR['noisy']['d_pred']


# ---------------------------------------------------------------------------
# model construction and host-side refusals (no GPU needed)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize('loss', ['ssim', 'l1', 'barron,1e+0ssim'])
def test_model_constructs_with_the_new_losses(loss):
    import losses
    import models
    from util import io as ioutil
    m = models.get_model_class('nlt')(ioutil.make_config(loss=loss, uvh=64, uvw=64, imh=64, imw=64))
    kinds = [type(f).__name__ for _, f in m.wloss]
    assert kinds == {'ssim': ['SSIM'], 'l1': ['L1'], 'barron,1e+0ssim': ['Barron', 'SSIM']}[loss]
    ssim = [f for _, f in m.wloss if isinstance(f, losses.SSIM)]
    assert all(f.dynamic_range == 1.0 for f in ssim)


def test_host_side_refusals():
    import losses
    import nlt_native as nat
    lib = nat.lib()
    x = torch.zeros(1, 10, 32, 3)
    with pytest.raises(ValueError):
        losses.SSIM(1)(x, x)
    with pytest.raises(ValueError):
        losses.SSIM(1)(x.transpose(1, 2).contiguous(), x.transpose(1, 2).contiguous())
    y = torch.zeros(1, 16, 16, 3)
    for f in (losses.SSIM(1), losses.L1()):
        with pytest.raises(NotImplementedError):
            f(y, y, weights=torch.ones(1, 16, 16, 1))
    assert lib.nlt_ssim_loss_workspace_bytes(1, 10, 11) < 0
    assert lib.nlt_ssim_loss_workspace_bytes(1, 11, 10) < 0
    assert lib.nlt_ssim_loss_workspace_bytes(0, 64, 64) < 0
    assert lib.nlt_ssim_loss_workspace_bytes(1, 11, 11) > 0
    assert lib.nlt_ssim_loss_workspace_bytes(32, 1024, 1024) >= 32 * 32 * 32 * 8
    assert lib.nlt_l1_loss_workspace_bytes(0, 12) < 0
    assert lib.nlt_l1_loss_workspace_bytes(2, 0) < 0
    assert lib.nlt_l1_loss_workspace_bytes(2, 12) > 0
    # argument validation happens before any CUDA call
    assert lib.nlt_ssim_loss(None, None, 1, 16, 16, 1.0, 1.0, None, None, None, None) < 0
    assert lib.nlt_l1_loss(None, None, 1, 12, 1.0, None, None, None, None) < 0
