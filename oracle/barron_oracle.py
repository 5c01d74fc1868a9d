"""CPU restatement of the reference's *training* loss term "barron" (SURVEY.md section 8f, row N1) -- TEST
INFRASTRUCTURE ONLY, like the rest of oracle/: nothing under neural-light-transport_b200/ may import it.

What the reference computes (nlt/losses.py:90-121): the residual `gt - pred` (alpha-blended when weights are
given) goes through robust_loss's `AdaptiveImageLossFunction` configured with color_space 'YUV', representation
'CDF9/7', 5 wavelet levels, scale base 1, and alpha / scale FIXED (alpha_lo == alpha_hi == 1, scale_lo ==
scale_init == 0.01), i.e. (third_party/robust_loss/adaptive.py:450-518, distribution.py:181-222, general.py:29-125):

    r   = rgb -> volume-preserving YUV              (util.py:97-115: 1.580227820074 * tf.image.rgb_to_yuv)
    w   = flatten(CDF 9/7 analysis of every channel, 5 levels, reflecting boundaries)   (wavelet.py:33-94,197-334,408-441)
    nll = sqrt((w / 0.01)^2 + 1) - 1  +  log(0.01)  +  log Z(1)                          (Charbonnier = general loss at alpha 1)

then the mean over everything but the batch axis (`keep_batch=True`) or over everything.

PINNED by the reference's own fixtures (tests/test_oracle_barron.py): the CDF 9/7 pyramid of
third_party/robust_loss/data/wavelet_golden.mat (an 83x71 RGB image decomposed by an independent implementation,
upstream tolerance 1e-5), the two `pad_reflecting` golden index vectors of wavelet_test.py:89-121, the knots of
partition_spline.npz around alpha = 1 (and the closed form log(2 e K_1(1)) they approximate to 1e-6).
Written in torch (float64 capable, differentiable) so that it can also serve as the gradient oracle of a future
CUDA implementation of this loss.
"""
import math

import torch

# tf.image.rgb_to_yuv's matrix (rows: R, G, B contributions to Y, U, V), times the constant that makes the map
# volume preserving (determinant 1): third_party/robust_loss/util.py:97-115
_YUV_FROM_RGB = ((0.299, -0.14714119, 0.61497538),
                 (0.587, -0.28886916, -0.51496512),
                 (0.114, 0.43601035, -0.10001026))
SYUV_SCALE = 1.580227820074

# Cohen-Daubechies-Feauveau 9/7 analysis filters, centre tap first (Cohen et al. 1992; wavelet.py:56-72)
_CDF97_LO_HALF = (0.852698679009, 0.377402855613, -0.110624404418, -0.023849465020, 0.037828455507)
_CDF97_HI_HALF = (0.788485616406, -0.418092273222, -0.040689417609, 0.064538882629)


def rgb_to_syuv(rgb):
    m = torch.tensor(_YUV_FROM_RGB, dtype=rgb.dtype, device=rgb.device)
    return SYUV_SCALE * (rgb @ m)


def _symmetric(half, dtype):
    h = torch.tensor(half, dtype=dtype)
    return torch.cat((h.flip(0)[:-1], h))       # [f(n-1) .. f(1) f(0) f(1) .. f(n-1)]


def cdf97_analysis_filters(dtype=torch.float64):
    return _symmetric(_CDF97_LO_HALF, dtype), _symmetric(_CDF97_HI_HALF, dtype)


def reflect_indices(n, below, above):
    """Source index of every element of a length-n axis padded by `below` / `above` entries with REFLECTING
    boundaries (edge sample not repeated), any number of reflections (wavelet.py:97-147)."""
    i = torch.arange(-below, n + above)
    period = max(1, 2 * (n - 1))
    r = torch.remainder(i, period)
    return torch.minimum(2 * (n - 1) - r, r) if n > 1 else torch.zeros_like(i)


def _filter_decimate(x, f, axis, shift):
    """Correlate [C, A, B] with the odd-length filter `f` along spatial axis `axis` (0 -> A, 1 -> B) under
    reflecting boundaries, after dropping `shift` leading padded samples, and keep every second output
    (wavelet.py:170-218)."""
    dim = axis + 1
    n = x.shape[dim]
    idx = reflect_indices(n, (len(f) - 1) // 2, len(f) // 2).to(x.device)
    xp = x.index_select(dim, idx)
    xp = xp.narrow(dim, shift, xp.shape[dim] - shift)
    win = xp.unfold(dim, len(f), 2)                       # [..., n_out, ..., taps]
    return (win * f.to(device=x.device, dtype=x.dtype)).sum(-1)


def wavelet_construct(im, num_levels):
    """im [C, A, B] -> ((hh, lh, hl) per level ..., residual), the band order of wavelet.py:293-334:
    band0 = highpass along both axes, band1 = lowpass(axis 0) then highpass(axis 1), band2 = highpass(axis 0)
    then lowpass(axis 1).  Highpass taps start one sample later (shift 1)."""
    if im.dim() != 3:
        raise ValueError('Expected `im` to have a rank of 3, but is of size {}'.format(tuple(im.shape)))
    if num_levels > max_num_levels(im.shape):
        raise ValueError('num_levels %d exceeds what size %s supports' % (num_levels, tuple(im.shape)))
    lo, hi = cdf97_analysis_filters(im.dtype)
    pyr = []
    for _ in range(num_levels):
        h = _filter_decimate(im, hi, 0, 1)
        l = _filter_decimate(im, lo, 0, 0)
        pyr.append((_filter_decimate(h, hi, 1, 1), _filter_decimate(l, hi, 1, 1), _filter_decimate(h, lo, 1, 0)))
        im = _filter_decimate(l, lo, 1, 0)
    pyr.append(im)
    return tuple(pyr)


def max_num_levels(shape):
    return int(math.ceil(math.log2(max(1, min(shape[1], shape[2])))))


def wavelet_flatten(pyr):
    """Pyramid -> one [C, A, B] tensor in the usual quadrant layout: residual top-left, band1 right of it, band2
    below it, band0 diagonal; applied from the coarsest level outwards (wavelet.py:408-441)."""
    flat = pyr[-1]
    for level in reversed(pyr[:-1]):
        top = torch.cat((flat, level[1]), dim=2)
        bottom = torch.cat((level[2], level[0]), dim=2)
        flat = torch.cat((top, bottom), dim=1)
    return flat


def charbonnier(x, scale):
    """General robust loss at alpha = 1 (general.py:96-122 with beta = |alpha - 2| = 1)."""
    return torch.sqrt((x / scale) ** 2 + 1.0) - 1.0


def partition_curve(alpha):
    """x-coordinate into the log-partition spline for 0 <= alpha < 4 (distribution.py:88-114)."""
    return (2.25 * alpha - 4.5) / (abs(alpha - 2.0) + 0.25) + alpha + 2.0


def hermite(t, v0, v1, m0, m1):
    """Cubic Hermite segment on t in [0, 1] (cubic_spline.py:27-97)."""
    t2, t3 = t * t, t * t * t
    h01 = -2.0 * t3 + 3.0 * t2
    h00 = 1.0 - h01
    h11 = t3 - t2
    h10 = h11 - t2 + t
    return v0 * h00 + v1 * h01 + m0 * h10 + m1 * h11


def log_partition(alpha, x_scale, knot_lo, values, tangents):
    """log Z(alpha) from the two spline knots around it: `values` / `tangents` hold knots knot_lo, knot_lo + 1 of
    partition_spline.npz, `x_scale` its knots-per-unit (distribution.py:150-179)."""
    x = partition_curve(alpha) * x_scale
    t = x - knot_lo
    assert 0.0 <= t <= 1.0, 'alpha outside the supplied spline segment'
    return hermite(t, values[0], values[1], tangents[0], tangents[1])


def log_partition_alpha1_closed_form():
    """Z(1) = integral exp(-(sqrt(x^2 + 1) - 1)) dx = 2 e K_1(1)."""
    from scipy.special import kv
    return math.log(2.0 * math.e * float(kv(1, 1.0)))


def image_nll(residual, log_z, scale=0.01, num_levels=5):
    """residual [N, H, W, 3] -> per-element negative log-likelihoods [N, H, W, 3] in the flattened wavelet layout
    (adaptive.py:450-518 with fixed alpha 1 and fixed scale)."""
    n, h, w, c = residual.shape
    x = rgb_to_syuv(residual)
    stack = x.permute(0, 3, 1, 2).reshape(n * c, h, w)
    flat = wavelet_flatten(wavelet_construct(stack, num_levels))
    mat = flat.reshape(n, c, h, w).permute(0, 2, 3, 1)
    return charbonnier(mat, scale) + math.log(scale) + log_z


def image_nll_abs_grad(residual, scale=0.01, num_levels=5, grad_scale=1.0):
    """Magnitude companion of d(grad_scale * sum image_nll(residual)) / d(residual): |M|^T |W|^T |g| in the residual's
    [N, H, W, 3] layout, with g = grad_scale * d charbonnier / dw per wavelet coefficient, |W| the analysis run with
    absolute filter taps and |M| the scaled YUV matrix with absolute entries.  Every product of the chain taken in
    magnitude, so a computed gradient's rounding error is a few units of its precision times this, wherever the
    signed sums cancel.  Multiply by |alpha| for an alpha-blended residual."""
    n, h, w, c = residual.shape
    stack = rgb_to_syuv(residual.detach()).permute(0, 3, 1, 2).reshape(n * c, h, w)
    with torch.no_grad():
        z = wavelet_flatten(wavelet_construct(stack, num_levels)) / scale
    g = (grad_scale / scale) * (z / torch.sqrt(z * z + 1.0)).abs()
    lo, hi = (f.abs() for f in cdf97_analysis_filters(residual.dtype))
    x0 = torch.zeros_like(stack, requires_grad=True)
    with torch.enable_grad():
        im, pyr = x0, []
        for _ in range(num_levels):         # wavelet_construct with |taps|
            hr = _filter_decimate(im, hi, 0, 1)
            lr = _filter_decimate(im, lo, 0, 0)
            pyr.append((_filter_decimate(hr, hi, 1, 1), _filter_decimate(lr, hi, 1, 1), _filter_decimate(hr, lo, 1, 0)))
            im = _filter_decimate(lr, lo, 1, 0)
        pyr.append(im)
        gx, = torch.autograd.grad(wavelet_flatten(tuple(pyr)), x0, g)
    m = SYUV_SCALE * torch.tensor(_YUV_FROM_RGB, dtype=residual.dtype, device=residual.device).abs()
    return gx.reshape(n, c, h, w).permute(0, 2, 3, 1) @ m.t()


def barron_loss(gt, pred, log_z, keep_batch=False, weights=None):
    """nlt/losses.py:108-121.  weights: alpha map broadcast over channels (util/img.py alpha_blend)."""
    if weights is not None:
        gt, pred = gt * weights, pred * weights
    nll = image_nll(gt - pred, log_z)
    return nll.mean(dim=(1, 2, 3)) if keep_batch else nll.mean()
