"""Losses with the reference's class names (nlt/losses.py).

L2 (SURVEY.md 8a a10: the loss used when timing the path), L1, SSIM and Barron (row N1:
the first term of the shipped `loss = barron,1e+0lpips`) are each fused with their own
gradient in CUDA.  LPIPS (the second term) raises NotImplementedError.
"""
import torch

import nlt_native as nat


class L2():
    """nlt/losses.py:39-53 -- mean squared error; keep_batch -> (N,)."""

    def __init__(self):
        self._ws = None
        self.d_pred = None      # gradient of sum_b(loss_b) * grad_scale w.r.t. pred
        self.grad_scale = None  # set by the train step: 1 / global_bs

    def __call__(self, gt, pred, keep_batch=False, weights=None):
        if weights is not None:
            raise NotImplementedError('sample weights')
        lib = nat.lib()
        B = pred.shape[0]
        per = pred.numel() // B
        need = lib.nlt_l2_loss_workspace_bytes(B, per)
        if self._ws is None or self._ws.numel() * 4 < need or self._ws.device != pred.device:
            self._ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=pred.device)
        loss = torch.empty(B, dtype=torch.float32, device=pred.device)
        want_grad = self.grad_scale is not None
        self.d_pred = torch.empty_like(pred) if want_grad else None
        scale = float(self.grad_scale) if want_grad else 0.0
        if not keep_batch and want_grad:
            scale = scale / B   # mean over the batch as well
        from engine import PROF
        PROF.run('fwd loss l2', 4 * pred.numel() * (3 if want_grad else 2), lambda: nat.check(lib.nlt_l2_loss(
            nat.ptr(pred), nat.ptr(gt), B, per, scale, nat.ptr(loss), nat.ptr(self.d_pred), nat.ptr(self._ws),
            nat.stream())))
        if keep_batch:
            return loss
        return loss.mean()


class L1():
    """nlt/losses.py:27-36 -- mean absolute error; keep_batch -> (N,), fused with its gradient (nlt_l1_loss).
    The reference's L1 takes no keep_batch (DESIGN.md section 1, difference (vi)); keep_batch=False gives its scalar."""

    def __init__(self):
        self._ws = None
        self.d_pred = None
        self.grad_scale = None

    def __call__(self, gt, pred, keep_batch=False, weights=None):
        if weights is not None:
            raise NotImplementedError('sample weights')
        lib = nat.lib()
        B = pred.shape[0]
        per = pred.numel() // B
        need = lib.nlt_l1_loss_workspace_bytes(B, per)
        if need < 0:
            nat.check(-1)
        if self._ws is None or self._ws.numel() * 4 < need or self._ws.device != pred.device:
            self._ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=pred.device)
        loss = torch.empty(B, dtype=torch.float32, device=pred.device)
        want_grad = self.grad_scale is not None
        self.d_pred = torch.empty_like(pred) if want_grad else None
        scale = float(self.grad_scale) if want_grad else 0.0
        if not keep_batch and want_grad:
            scale = scale / B
        from engine import PROF
        PROF.run('fwd loss l1', 4 * pred.numel() * (3 if want_grad else 2), lambda: nat.check(lib.nlt_l1_loss(
            nat.ptr(pred), nat.ptr(gt), B, per, scale, nat.ptr(loss), nat.ptr(self.d_pred), nat.ptr(self._ws),
            nat.stream())))
        return loss if keep_batch else loss.mean()


class SSIM():
    """nlt/losses.py:75-87 -- (1 - tf.image.ssim(gt, pred, dynamic_range)) / 2 per sample; keep_batch -> (N,), fused
    with its gradient (nlt_ssim_loss).  The reference's SSIM takes no keep_batch (DESIGN.md section 1, difference
    (vi)); keep_batch=False gives its scalar.  Images need at least 11 x 11 pixels (the window, VALID)."""
    WIN = 11

    def __init__(self, dynamic_range):
        self.dynamic_range = float(dynamic_range)
        self._ws = None
        self.d_pred = None
        self.grad_scale = None

    def __call__(self, gt, pred, keep_batch=False, weights=None):
        if weights is not None:
            raise NotImplementedError('sample weights')
        B, H, W, C3 = pred.shape
        if C3 != 3 or H < self.WIN or W < self.WIN or tuple(gt.shape) != tuple(pred.shape):
            raise ValueError('ssim: expected two [N, H >= %d, W >= %d, 3] images, got %s and %s' % (
                self.WIN, self.WIN, tuple(gt.shape), tuple(pred.shape)))
        lib = nat.lib()
        need = lib.nlt_ssim_loss_workspace_bytes(B, H, W)
        if need < 0:
            nat.check(-1)
        if self._ws is None or self._ws.numel() * 4 < need or self._ws.device != pred.device:
            self._ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=pred.device)
        loss = torch.empty(B, dtype=torch.float32, device=pred.device)
        want_grad = self.grad_scale is not None
        self.d_pred = torch.empty_like(pred) if want_grad else None
        scale = float(self.grad_scale) if want_grad else 0.0
        if not keep_batch and want_grad:
            scale = scale / B
        from engine import PROF
        PROF.run('fwd loss ssim', 4 * pred.numel() * (3 if want_grad else 2), lambda: nat.check(lib.nlt_ssim_loss(
            nat.ptr(pred), nat.ptr(gt), B, H, W, self.dynamic_range, scale, nat.ptr(loss), nat.ptr(self.d_pred),
            nat.ptr(self._ws), nat.stream())))
        return loss if keep_batch else loss.mean()


class Barron():
    """nlt/losses.py:90-121 -- the adaptive robust loss with FIXED alpha = 1 (Charbonnier) and scale = 0.01 on a
    5-level CDF 9/7 wavelet decomposition of the scaled-YUV residual; keep_batch -> (N,).  One fused CUDA call
    produces the per-sample losses and d(sum_b loss_b * grad_scale)/d(pred) (nlt_barron_loss).

    The arithmetic is checked on the CPU (tests/test_barron_core.py) and the kernels on hardware
    (tests/test_gpu_barron.py, tests/test_gpu_barron_census.py) against the oracle that is pinned to the reference's
    own wavelet fixtures.  The per-sample losses are deterministic."""
    LOG_Z_ALPHA1 = 1.1854952323491930      # log Z(1) = log(2 e K_1(1)); the reference's spline agrees to 1e-10
    SCALE = 0.01
    LEVELS = 5

    def __init__(self, imw, imh):
        self.imw, self.imh = imw, imh
        self._ws = None
        self.d_pred = None
        self.grad_scale = None

    def __call__(self, gt, pred, keep_batch=False, weights=None):
        lib = nat.lib()
        B, H, W, C3 = pred.shape
        if C3 != 3 or (H, W) != (self.imh, self.imw):
            raise ValueError('expected [N, %d, %d, 3] images, got %s' % (self.imh, self.imw, tuple(pred.shape)))
        need = lib.nlt_barron_loss_workspace_bytes(B, H, W, self.LEVELS)
        if need < 0:
            nat.check(-1)
        if self._ws is None or self._ws.numel() * 4 < need or self._ws.device != pred.device:
            self._ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=pred.device)
        loss = torch.empty(B, dtype=torch.float32, device=pred.device)
        want_grad = self.grad_scale is not None
        self.d_pred = torch.empty_like(pred) if want_grad else None
        scale = float(self.grad_scale) if want_grad else 0.0
        if not keep_batch and want_grad:
            scale = scale / B
        if weights is not None:
            weights = weights.to(pred.device, torch.float32).expand(B, H, W, 1).contiguous()
        from engine import PROF
        PROF.run('fwd loss barron', 4 * pred.numel() * (3 if want_grad else 2), lambda: nat.check(lib.nlt_barron_loss(
            nat.ptr(pred), nat.ptr(gt), nat.ptr(weights), B, H, W, self.LEVELS, self.SCALE, self.LOG_Z_ALPHA1, scale,
            nat.ptr(loss), nat.ptr(self.d_pred), nat.ptr(self._ws), nat.stream())))
        return loss if keep_batch else loss.mean()


class LPIPS():
    def __init__(self, per_ch=False):
        raise NotImplementedError('lpips: next row N1 (SURVEY.md 8f)')
