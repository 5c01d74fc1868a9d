"""fp64 oracles of the L1 and SSIM training losses.  TEST INFRASTRUCTURE ONLY, like oracle/nlt_oracle.py.

Restatements, in plain PyTorch ops, of the reference's `losses.L1` and `losses.SSIM` (nlt/losses.py:27-36, 75-87) and
of the TF 2.2 routines behind `tf.image.ssim` (image_ops_impl `_fspecial_gauss`, `_ssim_helper`,
`_ssim_per_channel`).  TensorFlow cannot be installed offline, so these are not compared with TF itself: they are
pinned by the CPU tests (tests/test_oracle_losses.py: the window's definition, known answers, an independent scipy
restatement, gradcheck).
"""
import torch
import torch.nn.functional as F

def l1_loss(gt, pred, keep_batch=False):
    """losses.L1 -- nlt/losses.py:27-36: tf.keras.losses.MeanAbsoluteError(reduction='none') averages |gt - pred| over
    the last axis, then tf.reduce_mean.  keep_batch -> (N,) is this project's per-sample form (the reference's L1
    has no keep_batch); the scalar is the mean of the per-sample values, all samples having the same size.  The
    gradient of |.| at a tie is 0, as TF's Abs gradient (sign)."""
    ae = (gt - pred).abs().mean(dim=-1)
    return ae.mean(dim=(1, 2)) if keep_batch else ae.mean()


SSIM_FILTER_SIZE, SSIM_FILTER_SIGMA, SSIM_K1, SSIM_K2 = 11, 1.5, 0.01, 0.03   # tf.image.ssim defaults (TF 2.2)


def fspecial_gauss(size=SSIM_FILTER_SIZE, sigma=SSIM_FILTER_SIGMA, dtype=torch.float64):
    """_fspecial_gauss of TF 2.2 image_ops_impl: coords = arange(size) - (size - 1) / 2; g = coords^2 * (-0.5 / sigma^2);
    g = g[None, :] + g[:, None]; softmax over the flattened window -> [size, size]."""
    coords = torch.arange(size, dtype=dtype) - (size - 1) / 2.0
    g = coords ** 2 * (-0.5 / sigma ** 2)
    g = g.reshape(1, -1) + g.reshape(-1, 1)
    return torch.softmax(g.reshape(1, -1), dim=-1).reshape(size, size)


def ssim_terms(gt, pred, max_val=1.0):
    """_ssim_helper of TF 2.2 (compensation 1) with the depthwise VALID reducer of _ssim_per_channel, on [N,H,W,C]
    images: returns the luminance and contrast-structure maps [N, C, H - 10, W - 10]."""
    n, h, w, c = gt.shape
    if h < SSIM_FILTER_SIZE or w < SSIM_FILTER_SIZE:
        raise ValueError('ssim: images must be at least %d x %d, got %d x %d' % (SSIM_FILTER_SIZE, SSIM_FILTER_SIZE, h, w))
    kernel = fspecial_gauss(dtype=gt.dtype).to(gt.device).expand(c, 1, SSIM_FILTER_SIZE, SSIM_FILTER_SIZE)

    def reducer(t):        # depthwise_conv2d(t, kernel, strides=[1, 1, 1, 1], padding='VALID')
        return F.conv2d(t, kernel, groups=c)

    x, y = gt.permute(0, 3, 1, 2), pred.permute(0, 3, 1, 2)
    c1, c2 = (SSIM_K1 * max_val) ** 2, (SSIM_K2 * max_val) ** 2
    mean0, mean1 = reducer(x), reducer(y)
    num0 = mean0 * mean1 * 2.0
    den0 = mean0 ** 2 + mean1 ** 2
    luminance = (num0 + c1) / (den0 + c1)
    num1 = reducer(x * y) * 2.0
    den1 = reducer(x ** 2 + y ** 2)
    cs = (num1 - num0 + c2) / (den1 - den0 + c2)
    return luminance, cs


def ssim(gt, pred, max_val=1.0):
    """tf.image.ssim(gt, pred, max_val): mean of luminance * cs over the valid pixels ([-3, -2]), then the channels."""
    luminance, cs = ssim_terms(gt, pred, max_val)
    return (luminance * cs).mean(dim=(2, 3)).mean(dim=1)


def ssim_loss(gt, pred, max_val=1.0, keep_batch=False):
    """losses.SSIM -- nlt/losses.py:75-87: (1 - tf.image.ssim(gt, pred, dynamic_range)) / 2, then reduce_mean.
    keep_batch -> (N,) is this project's per-sample form (the reference's SSIM has no keep_batch)."""
    loss = (1 - ssim(gt, pred, max_val)) / 2
    return loss if keep_batch else loss.mean()
