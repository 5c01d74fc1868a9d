"""Op-level parity: every CUDA entry point of include/nlt_b200.h against the
oracle on seeded inputs.  Tolerances are fp32 round-off of sums of K terms
(the SIMT path is plain fp32 FMA; no tensor-core truncation)."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nlt_oracle as O   # noqa: E402


def _mods():
    import engine
    import nlt_native as nat
    return engine, nat


def _close(got, want, rtol=2e-5, atol=2e-5):
    got = got.detach().double().cpu().numpy()
    want = want.detach().double().cpu().numpy()
    scale = max(1.0, float(np.abs(want).max()))
    np.testing.assert_allclose(got, want, rtol=rtol, atol=atol * scale)


GEOMS = [
    # kind, k, s, H, W, seg channels, cout
    ('conv', 1, 1, 8, 8, [3, 1, 1], 16),
    ('conv', 1, 1, 16, 8, [4, 32], 3),
    ('conv', 2, 2, 16, 16, [16, 16], 16),
    ('conv', 2, 1, 8, 8, [16], 16),
    ('conv', 2, 2, 8, 8, [32, 32], 64),
    ('conv', 2, 1, 4, 4, [256], 256),
    ('conv', 3, 1, 9, 7, [5], 8),
    ('conv', 3, 2, 8, 8, [8, 4], 32),
    ('conv', 3, 2, 7, 9, [6], 12),
    ('conv', 4, 2, 8, 8, [16], 20),
    ('conv', 2, 2, 2, 2, [512, 512], 128),
    ('deconv', 2, 2, 4, 4, [64, 64, 64, 64], 128),
    ('deconv', 2, 1, 8, 8, [128], 128),
    ('deconv', 2, 2, 8, 8, [8, 32], 4),
    ('deconv', 2, 1, 16, 16, [4], 4),
    ('deconv', 3, 2, 5, 6, [16, 3], 8),
    ('deconv', 3, 1, 6, 5, [7], 5),
    ('deconv', 4, 2, 4, 4, [16], 16),
    ('deconv', 1, 2, 4, 4, [8], 8),
    ('deconv', 2, 2, 1, 1, [1024, 1024], 64),
    # pointwise kernel (1x1, <=64 -> <=16 channels), incl. the final conv's dgrad shape
    ('conv', 1, 1, 16, 16, [4, 16, 16], 3),
    ('conv', 1, 1, 8, 8, [36], 8),
    ('conv', 1, 1, 8, 8, [64], 16),
    # k == s transposed with Cout % 4 != 0: phase path instead of depth-to-space
    ('deconv', 2, 2, 4, 4, [8], 3),
    ('conv', 2, 2, 8, 8, [6, 3], 16),
    # enough pixels for the persistent CTAs to walk several tiles each
    ('conv', 2, 2, 512, 512, [16], 16),
    ('deconv', 2, 2, 128, 256, [8, 32], 4),
    ('conv', 2, 1, 256, 256, [16], 16),
    ('deconv', 2, 2, 64, 64, [32, 64], 32),
    # tensor-core (wgmma, 3xTF32) eligible shapes: every source C % 32 == 0, Cout % 16 == 0, tileable lattice
    ('conv', 2, 2, 32, 32, [32, 32], 64),       # patch view (5-D TMA), lattice 16x16 -> tile 8x16
    ('conv', 2, 1, 16, 16, [64], 64),           # stride-1 taps, SAME pad by TMA OOB fill
    ('conv', 3, 1, 16, 16, [32], 32),           # negative start coordinates
    ('deconv', 2, 2, 16, 16, [64, 64], 32),     # depth-to-space, N' = 128
    ('deconv', 2, 1, 16, 16, [32], 32),
    ('conv', 2, 2, 64, 256, [32], 128),         # lattice width 128 -> tile 1x128
    ('conv', 2, 1, 32, 32, [256], 256),         # two column tiles of 128, K = 1024
    ('deconv', 2, 2, 16, 16, [128, 128], 128),  # N' = 512: four column tiles
    ('conv', 1, 1, 16, 16, [64, 32], 48),       # BN = 16
    # 16-channel sources: 64-byte rows / SWIZZLE_64B K-blocks
    ('conv', 2, 2, 32, 32, [16, 16], 16),       # level-1 query conv shape
    ('conv', 2, 1, 16, 16, [16], 16),
    ('deconv', 2, 2, 16, 16, [16, 32, 32], 8),  # level-11 up-conv shape: N' = 32
    # row-run weight-gradient kernel: runs of 64 lattice pixels, ragged last run, SAME padding on both sides
    ('conv', 2, 1, 8, 72, [16], 16),
    ('conv', 3, 1, 9, 70, [8], 8),
    ('deconv', 2, 2, 8, 40, [8, 32], 4),
    ('conv', 2, 2, 6, 200, [16, 16], 16),
    ('deconv', 2, 1, 32, 16, [16], 16),
    ('conv', 2, 2, 64, 64, [32, 16], 32),       # mixed 32/16 sources -> 16-wide blocks
    # wide pointwise conv into 16 channels (nlt_pwx.cu: level 0 of the 64-channel query stack): cp.async-staged
    # 256-pixel tiles, ragged last tile, float4-able and scalar sources mixed, K not a multiple of 32.
    # The depth-to-space input gradients of the next five shapes run on pwd2s_mma_kernel (tc = 1 and pwmma = 1, the
    # defaults) and on pwd2s_kernel with tc = 0 or pwmma = 0
    ('conv', 2, 2, 8, 512, [16, 16], 32),       # its input gradients: depth-to-space K = 32 -> 4 x 16
    ('conv', 2, 2, 16, 256, [32], 64),          # 32-channel sources (pwd2s_kernel: two threads per pixel), K = 64
    ('conv', 2, 2, 32, 128, [32, 32], 64),      # ... lattice rows narrower than a tile: two rows per tile
    ('conv', 2, 2, 32, 128, [16], 16),          # ... four lattice rows per tile, 16-channel source
    ('conv', 2, 2, 32, 128, [32], 32),          # K = 32 -> 4 x 32
    # staged-patch weight gradient of the 2x2 convs (pws_wgrad_kernel): all four lane layouts, both strides,
    # SAME padding at the right / bottom edge
    ('conv', 2, 2, 16, 256, [16, 16], 16),      # K = 128, N = 16
    ('conv', 2, 1, 8, 128, [16], 32),           # K = 64, N = 32, stride 1
    ('conv', 2, 1, 8, 64, [32], 32),            # K = 128, N = 32 (two warps share a pixel's K rows), stride 1
    ('conv', 2, 1, 5, 192, [16], 16),           # K = 64, N = 16, stride 1, three tiles per row
    # row-stream stencil kernel (nlt_tiny.cu): 4 / 8 / 16 channels, ragged last tile, SAME padding either side
    ('deconv', 2, 1, 12, 200, [4], 4),
    ('deconv', 2, 1, 9, 128, [8], 8),
    ('conv', 2, 1, 7, 130, [8], 8),
    ('deconv', 2, 1, 6, 96, [16], 16),
    ('conv', 2, 1, 6, 64, [4], 4),
    # staged-patch forward of the stride-2 2x2 convs (pf_fwd_kernel): K = 64 / 128 into 16 / 32 channels
    ('conv', 2, 2, 4, 512, [16], 32),
    ('conv', 2, 2, 4, 256, [32], 16),
    ('conv', 2, 2, 6, 256, [16, 16], 32),
    # register-tile outer-product weight gradient (nlt_wop.cu), up-conv into 16 channels: 16 warps per CTA
    ('deconv', 2, 2, 4, 64, [32, 64, 64], 16),
    ('deconv', 2, 2, 5, 48, [16], 16),
    # ... and the same kernel as the input gradient of up-convs (patch K = 16 / 32 / 64 of the gradient, + beta, mask)
    ('deconv', 2, 2, 2, 128, [32], 16),
    # depth-to-space forward of the up-convs into 4 / 8 channels (pwx_d2s_fwd_kernel): 128-pixel row tiles
    ('deconv', 2, 2, 3, 128, [8, 32], 4),
    ('deconv', 2, 2, 2, 256, [16, 32, 32], 8),
    ('deconv', 2, 2, 2, 128, [4, 20], 4),
    ('deconv', 2, 2, 2, 128, [8, 28], 8),       # K = 36: zero-padded to 40 columns
    ('conv', 1, 1, 33, 37, [3, 60, 1], 16),
    ('conv', 1, 1, 32, 32, [64], 16),
    ('conv', 1, 1, 24, 24, [20, 4], 16),
    ('conv', 1, 1, 40, 40, [3, 40, 1, 2], 16),
    ('conv', 1, 1, 24, 40, [32, 40, 8], 16),
    # coalesced weight gradient of a 1x1 conv into <= 4 channels (wopn_wgrad_kernel: >= 64 K pixels)
    ('conv', 1, 1, 160, 144, [4, 16, 16], 3),
    ('conv', 1, 1, 128, 192, [8, 32], 2),    # K = 80: 24 float4 groups per row (forward at 51 KB, weight gradient at 67 KB)
]


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', GEOMS)
@pytest.mark.parametrize('act', ['leakyrelu', None, 'relu'])
def test_gconv_forward_backward(kind, k, s, H, W, segc, cout, act):
    engine, nat = _mods()
    torch.manual_seed(hash((kind, k, s, H, W, cout)) % 1000)
    N = 3
    dev = torch.device('cuda')
    xs = [torch.randn(N, H, W, c) for c in segc]
    layer = engine.ConvLayer(kind, k, s, cout, act)
    layer.build(sum(segc), dev, torch.Generator().manual_seed(1))
    layer.bias.copy_(torch.randn(cout) * 0.1)
    # oracle (fp64)
    w64 = layer.kernel.double().cpu().requires_grad_(True)
    b64 = layer.bias.double().cpu().requires_grad_(True)
    x64 = [x.double().requires_grad_(True) for x in xs]
    fn = O.conv2d_same if kind == 'conv' else O.conv2d_transpose_same
    y64 = fn(torch.cat(x64, dim=3), w64, b64, s)
    if act:
        y64 = O.act(y64, act)
    # product
    tape = engine.Tape()
    acts = [engine.Act(x.to(dev).contiguous(), act='leakyrelu', needs_grad=True) for x in xs]
    y = layer.forward([engine.Seg(a) for a in acts], tape)
    _close(y.t, y64)
    gy = torch.randn_like(y64)
    y64.backward(gy)
    # dz is what the tape expects in y.grad (mask of y's own activation applied by its producer)
    dz64 = gy * (torch.where(y64 > 0, 1.0, 0.3) if act == 'leakyrelu' else
                 torch.where(y64 > 0, 1.0, 0.0) if act == 'relu' else 1.0)
    y.grad = dz64.float().to(dev).contiguous()
    tape.backward()
    _close(layer.gkernel, w64.grad, rtol=1e-4, atol=1e-4)
    _close(layer.gbias, b64.grad, rtol=1e-4, atol=1e-4)
    for a, x in zip(acts, x64):
        # every input Act was declared as a leakyrelu output: its grad carries the mask of a.t
        want = x.grad * torch.where(x > 0, 1.0, 0.3)
        _close(a.grad, want, rtol=1e-4, atol=1e-4)


WOP_ALL_SHAPES = [g for g in GEOMS if g[4] >= 32 and (
    (g[0] == 'deconv' and g[1] == 2 and g[2] == 2 and g[6] in (4, 8, 16) and all(c % 4 == 0 for c in g[5])) or
    (g[1] == 2 and g[2] == 1 and g[5] == [16] and g[6] == 16))]


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', WOP_ALL_SHAPES)
def test_outer_product_wgrad_all_shapes(kind, k, s, H, W, segc, cout):
    """nlt_wop.cu also serves the up-convs and the 16 -> 16 stencils (option wop = 2; off by default because the
    staged-patch / wgmma kernels are faster there): same oracle check as every other route."""
    import nlt_native as nat
    with nat.options(wop=2):
        test_gconv_forward_backward(kind, k, s, H, W, segc, cout, 'leakyrelu')


NS2_SHAPES = [g for g in GEOMS if g[6] in (16, 32) and g[4] >= 128 and (
    (g[0] == 'conv' and g[1] == 1) or (g[1] == 2 and g[2] == 2))][:12] + [('conv', 1, 1, 32, 32, [64], 16)]


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', NS2_SHAPES)
def test_two_threads_per_pixel_forward_kernels(kind, k, s, H, W, segc, cout):
    """The pointwise / staged-patch forward kernels also exist with two threads per pixel (options pwx_ns / pf_ns = 2,
    off by default): same oracle check."""
    import nlt_native as nat
    with nat.options(pwx_ns=2, pf_ns=2, pf=1):
        test_gconv_forward_backward(kind, k, s, H, W, segc, cout, 'leakyrelu')


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', [('conv', 2, 2, 4, 512, [16], 32), ('conv', 2, 2, 4, 256, [32], 16),
                                                    ('conv', 2, 2, 6, 256, [16, 16], 16), ('conv', 2, 2, 16, 256, [32], 64),
                                                    ('conv', 2, 2, 32, 128, [32, 32], 64)])
def test_staged_patch_forward_and_pwd2s_first_routes(kind, k, s, H, W, segc, cout):
    """Options pf (staged-patch forward of the 2x2/s2 convs) and pwd2s_first (depth-to-space input gradient ahead of
    the tensor path for 64-channel gradients), both off by default: same oracle check on the routes they select, and
    the kernel of the route must have run (K = 64 / 128 forwards into 16 / 32 channels: pf_fwd_kernel; input gradients
    into 16- / 32-channel sources: pwd2s_kernel)."""
    import nlt_native as nat
    kernel = 'pf_fwd_kernel' if H in (4, 6) else 'pwd2s_kernel'
    with nat.options(pf=1, pwd2s_first=1):
        n0 = nat.kernel_launch_count(kernel)
        test_gconv_forward_backward(kind, k, s, H, W, segc, cout, 'leakyrelu')
        assert nat.kernel_launch_count(kernel) > n0, kernel + ' did not run'


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', [('conv', 2, 1, 5, 128, [16], 16), ('deconv', 2, 1, 5, 256, [16], 16),
                                                    ('conv', 2, 1, 256, 256, [16], 16)])
def test_staged_patch_kernel_on_stride1_stencils(kind, k, s, H, W, segc, cout):
    """pf_fwd_kernel in its stride-1 form (option pf_s1): forward and input gradient of the 16 -> 16 2x2 stencils,
    SAME padding on either side (conv / deconv flavour)."""
    import nlt_native as nat
    with nat.options(pf_s1=1, pf=1):
        for act in ('leakyrelu', None):
            n0 = nat.kernel_launch_count('pf_fwd_kernel')
            test_gconv_forward_backward(kind, k, s, H, W, segc, cout, act)
            assert nat.kernel_launch_count('pf_fwd_kernel') > n0, 'pf_fwd_kernel did not run'


TC_SHAPES = [g for g in GEOMS if all(c % 16 == 0 for c in g[5]) and g[6] % 16 == 0 and g[3] * g[4] >= 256]


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', [g for g in GEOMS if all(c % 16 == 0 for c in g[5]) and g[6] % 16 == 0
                                                    and g[3] * g[4] >= 256][:14])
def test_tensor_core_raw_hi_operand(kind, k, s, H, W, segc, cout):
    """Option tc_rawhi: the hi operand is the activation truncated to TF32 (lo = x - trunc(x), exact before its own
    rounding) or, with 0, rounded to TF32.  Same oracle check, same tolerance for both splits; option tc = 2 puts every
    shape on the wgmma kernel, and its launch counter must move."""
    import nlt_native as nat
    for v in (1, 0):         # default form, and the one that rounds hi
        with nat.options(tc=2, tc_rawhi=v):
            n0 = nat.tc_launch_count()
            test_gconv_forward_backward(kind, k, s, H, W, segc, cout, 'leakyrelu')
            assert nat.tc_launch_count() > n0, 'tensor-core kernel did not run'


@pytest.fixture(params=['ss', 'ts'])
def tc_form(request):
    """Both forms of the wgmma forward / input-gradient kernel: 'ss' = hi / lo activation planes written to shared
    memory (both operands from shared memory), 'ts' = the activation operand split in registers (wgmma RS form)."""
    import nlt_native as nat
    with nat.options(tcs=1 if request.param == 'ts' else 0):
        yield request.param


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', TC_SHAPES)
def test_tensor_core_vs_fp32_kernels(kind, k, s, H, W, segc, cout, tc_form):
    """A/B on identical inputs: wgmma 3xTF32 kernels (forward, input gradients with beta + mask, weight /
    bias gradients) against the fp32-FMA kernels of the same library: relative Frobenius error <= 5e-6.  The tensor-core
    arm runs with option tc = 2, so that every shape the wgmma kernel can run takes it, whatever the size heuristics
    would pick in production."""
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(3)
    N = 2
    xs = [torch.randn(N, H, W, c, device=dev) for c in segc]
    dzs = None
    res = {}
    for mode in ('tc', 'fp32'):
        with nat.options(tc=2 if mode == 'tc' else 0):
            L = engine.ConvLayer(kind, k, s, cout, 'leakyrelu')
            L.build(sum(segc), dev, torch.Generator().manual_seed(1))
            L.bias.copy_(torch.linspace(-0.1, 0.1, cout, device=dev))
            acts = [engine.Act(x, act='leakyrelu', needs_grad=True) for x in xs]
            tape = engine.Tape()
            t0 = nat.tc_launch_count()
            y = L.forward([engine.Seg(a) for a in acts], tape)
            if dzs is None:
                dzs = torch.randn_like(y.t)
            y.grad = dzs.clone()
            tape.backward()
            res[mode] = dict(y=y.t.clone(), gk=L.gkernel.clone(), gb=L.gbias.clone(),
                             gx=[a.grad.clone() for a in acts], tc=nat.tc_launch_count() - t0)
    assert res['fp32']['tc'] == 0
    assert res['tc']['tc'] > 0
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    assert rel(res['tc']['y'], res['fp32']['y']) <= 1e-5      # 3xTF32: ~1e-6 per product, grows ~sqrt(K)
    # weight / bias gradients sum over every pixel: both paths carry fp32 accumulation error of their own
    assert rel(res['tc']['gk'], res['fp32']['gk']) <= 2e-5
    assert rel(res['tc']['gb'], res['fp32']['gb']) <= 2e-5
    for a, b in zip(res['tc']['gx'], res['fp32']['gx']):
        assert rel(a, b) <= 1e-5


ROWS_SHAPES = [g for g in GEOMS if all(c % 4 == 0 for c in g[5]) and g[6] % 4 == 0 and g[6] <= 16]


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', ROWS_SHAPES)
def test_wgrad_row_run_vs_flat_pixel_kernel(kind, k, s, H, W, segc, cout):
    """A/B on identical inputs: the row-run warp-stream weight-gradient kernel against the flat-pixel form of
    the same library (option "wgrad_rows"); both accumulate in fp32 in different orders."""
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(11)
    N = 3
    xs = [torch.randn(N, H, W, c, device=dev) for c in segc]
    dzs = None
    res = {}
    for mode in (1, 0):
        with nat.options(tc=0, wgrad_rows=mode):
            L = engine.ConvLayer(kind, k, s, cout, 'leakyrelu')
            L.build(sum(segc), dev, torch.Generator().manual_seed(1))
            acts = [engine.Act(x, act='leakyrelu', needs_grad=True) for x in xs]
            tape = engine.Tape()
            y = L.forward([engine.Seg(a) for a in acts], tape)
            if dzs is None:
                dzs = torch.randn_like(y.t)
            y.grad = dzs.clone()
            tape.backward()
            res[mode] = (L.gkernel.clone(), L.gbias.clone())
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    assert rel(res[1][0], res[0][0]) <= 1e-5
    assert rel(res[1][1], res[0][1]) <= 1e-5


@pytest.mark.parametrize('H,W,c_skip,c_other,down_cout,dk', [
    (16, 16, 16, 4, 16, 2), (8, 24, 16, 8, 32, 2), (6, 10, 12, 4, 8, 2),   # depth-to-space dgrad: shuffle / per-quad modes
    (8, 8, 16, 4, 16, 1), (4, 12, 8, 4, 24, 1),                             # 1x1 consumer: same-pixel mode
    (8, 512, 16, 4, 16, 2), (4, 1024, 16, 4, 32, 2)])                       # lattice rows of 256 / 512: the streaming pwd2s kernel (K = 16 / 32)
def test_final_conv_input_gradient_rides_on_down_conv_dgrad(H, W, c_skip, c_other, down_cout, dk):
    """Skip tensor consumed by a 2x2/s2 down-conv and, later, by the final 1x1 conv -> 3 (the level-0 skip
    of the network): with fusion on, the 1x1 conv's input gradient is added in the epilogue of the
    down-conv's input-gradient launch (nlt_gconv_fwd_fused).  Same result as the unfused engine and as
    autograd (fp64), one launch less, parameter gradients untouched."""
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(21)
    N = 2
    x_skip = torch.randn(N, H, W, c_skip, device=dev)
    x_other = torch.randn(N, H, W, c_other, device=dev)
    gen = lambda: torch.Generator().manual_seed(4)
    res = {}
    for fuse in (True, False):
        engine.FUSE_POINTWISE_DGRAD = fuse
        try:
            down = engine.ConvLayer('conv', dk, dk, down_cout, 'leakyrelu')
            down.build(c_skip, dev, gen())
            final = engine.ConvLayer('conv', 1, 1, 3, None)
            final.build(c_other + c_skip, dev, gen())
            a_skip = engine.Act(x_skip, act='leakyrelu', needs_grad=True)
            a_other = engine.Act(x_other, act='leakyrelu', needs_grad=True)
            tape = engine.Tape()
            y_down = down.forward([engine.Seg(a_skip)], tape)
            y_fin = final.forward([engine.Seg(a_other), engine.Seg(a_skip)], tape)
            torch.manual_seed(5)
            y_down.grad = torch.randn_like(y_down.t)
            y_fin.grad = torch.randn_like(y_fin.t)
            g_down, g_fin = y_down.grad.clone(), y_fin.grad.clone()
            n0 = nat.launch_count()
            tape.backward()
            res[fuse] = dict(gs=a_skip.grad.clone(), go=a_other.grad.clone(), gk=[down.gkernel.clone(), final.gkernel.clone()],
                             launches=nat.launch_count() - n0)
        finally:
            engine.FUSE_POINTWISE_DGRAD = True
    # fp64 autograd of the same graph
    xs64 = x_skip.double().cpu().requires_grad_(True)
    xo64 = x_other.double().cpu().requires_grad_(True)
    # y.grad handed to the tape is the gradient of the PRE-activation output (see test_gconv_forward_backward)
    pre = O.conv2d_same(xs64, down.kernel.double().cpu(), down.bias.double().cpu(), dk)
    yf = O.conv2d_same(torch.cat([xo64, xs64], -1), final.kernel.double().cpu(), final.bias.double().cpu(), 1)
    loss = (pre * g_down.double().cpu()).sum() + (yf * g_fin.double().cpu()).sum()
    loss.backward()
    want_s = xs64.grad * torch.where(xs64 > 0, 1.0, 0.3)
    want_o = xo64.grad * torch.where(xo64 > 0, 1.0, 0.3)
    for fuse in (True, False):
        _close(res[fuse]['gs'], want_s, rtol=1e-4, atol=1e-4)
        _close(res[fuse]['go'], want_o, rtol=1e-4, atol=1e-4)
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    assert rel(res[True]['gs'], res[False]['gs']) <= 1e-6
    assert rel(res[True]['go'], res[False]['go']) <= 1e-6
    for a, b in zip(res[True]['gk'], res[False]['gk']):
        assert torch.equal(a, b)
    if c_skip % 4 == 0:
        assert res[True]['launches'] == res[False]['launches'] - 1, (res[True]['launches'], res[False]['launches'])


@pytest.mark.parametrize('mode', [1, 2])
@pytest.mark.parametrize('kind,k,s,H,W,cin', [('conv', 2, 1, 16, 24, 32), ('conv', 2, 2, 32, 16, 16),
                                              ('conv', 2, 2, 16, 16, 32), ('deconv', 2, 1, 12, 20, 32),
                                              ('conv', 3, 1, 9, 11, 12)])
def test_wide_stencil_32_outputs(kind, k, s, H, W, cin, mode):
    """The 32-output form of the wide stencil kernel (option
    "dconv_wide32": 1 = one pixel per thread, 2 = two) against the default routing, fp32 kernels only."""
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(31)
    x = torch.randn(3, H, W, cin, device=dev)
    res = {}
    for m in (mode, 0):
        with nat.options(tc=0, dconv_wide32=m):
            L = engine.ConvLayer(kind, k, s, 32, 'leakyrelu')
            L.build(cin, dev, torch.Generator().manual_seed(1))
            L.bias.copy_(torch.linspace(-0.1, 0.1, 32, device=dev))
            a = engine.Act(x, act='leakyrelu', needs_grad=True)
            tape = engine.Tape()
            y = L.forward([engine.Seg(a)], tape)
            torch.manual_seed(5)
            y.grad = torch.randn_like(y.t)
            tape.backward()
            res[m] = (y.t.clone(), a.grad.clone(), L.gkernel.clone())
    rel = lambda p, q: float((p.double() - q.double()).norm() / q.double().norm())
    assert rel(res[mode][0], res[0][0]) <= 1e-5
    assert rel(res[mode][1], res[0][1]) <= 1e-5
    assert torch.equal(res[mode][2], res[0][2])          # weight gradients do not go through this kernel


@pytest.mark.parametrize('kind,k,s,H,W,cin', [('conv', 2, 2, 16, 24, 4), ('conv', 2, 2, 32, 16, 8), ('conv', 2, 1, 9, 16, 8),
                                              ('deconv', 2, 1, 12, 8, 8)])
def test_wide_stencil_preferred_over_quad_kernel(kind, k, s, H, W, cin):
    """Routing option "dconv_wide_first" (default on since round 2): 16 outputs from K <= 32 through the validated wide
    stencil kernel instead of the quad-per-thread kernel -- same results."""
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(33)
    x = torch.randn(3, H, W, cin, device=dev)
    res = {}
    for m in (1, 0):
        with nat.options(tc=0, dconv_wide_first=m):
            L = engine.ConvLayer(kind, k, s, 16, 'leakyrelu')
            L.build(cin, dev, torch.Generator().manual_seed(1))
            a = engine.Act(x, act='leakyrelu', needs_grad=True)
            tape = engine.Tape()
            y = L.forward([engine.Seg(a)], tape)
            torch.manual_seed(5)
            y.grad = torch.randn_like(y.t)
            tape.backward()
            res[m] = (y.t.clone(), a.grad.clone())
    rel = lambda p, q: float((p.double() - q.double()).norm() / q.double().norm())
    assert rel(res[1][0], res[0][0]) <= 1e-5 and rel(res[1][1], res[0][1]) <= 1e-5


@pytest.mark.parametrize('kind,k,s,H,W,segc,cout', [('conv', 2, 1, 16, 24, [8], 8), ('deconv', 2, 1, 12, 20, [8], 8),
                                                    ('conv', 2, 2, 16, 16, [4], 8), ('conv', 2, 2, 16, 16, [16, 16], 32),
                                                    ('conv', 2, 1, 9, 13, [8, 4], 8)])
def test_wide_stencil_8_outputs_and_virtual_concats(kind, k, s, H, W, segc, cout):
    """The 8-output form (options "dconv_wide8" + "dconv_wide_first") and virtual-concat sources of
    the wide routes, against the tiled / quad-per-thread routing."""
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(35)
    xs = [torch.randn(3, H, W, c, device=dev) for c in segc]
    res = {}
    for m in (1, 0):
        with nat.options(tc=0, dconv_wide8=m, dconv_wide32=m, dconv_wide_first=m):
            L = engine.ConvLayer(kind, k, s, cout, 'leakyrelu')
            L.build(sum(segc), dev, torch.Generator().manual_seed(1))
            acts = [engine.Act(x, act='leakyrelu', needs_grad=True) for x in xs]
            tape = engine.Tape()
            y = L.forward([engine.Seg(a) for a in acts], tape)
            torch.manual_seed(5)
            y.grad = torch.randn_like(y.t)
            tape.backward()
            res[m] = [y.t.clone()] + [a.grad.clone() for a in acts]
    rel = lambda p, q: float((p.double() - q.double()).norm() / q.double().norm())
    for p, q in zip(res[1], res[0]):
        assert rel(p, q) <= 1e-5


def test_tensor_core_path_is_taken_and_matches_fp32_path():
    """Eligible shapes must run on the wgmma kernel (launch counter moves) and agree with the
    fp32-FMA kernel of the same library to 3xTF32 accuracy (<= 4e-6 relative to the output scale)."""
    import ctypes as C
    engine, nat = _mods()
    dev = torch.device('cuda')
    lib = nat.lib()
    torch.manual_seed(5)
    x = [torch.randn(2, 32, 32, 32, device=dev), torch.randn(2, 32, 32, 32, device=dev)]
    L = engine.ConvLayer('conv', 2, 2, 64, 'leakyrelu')
    L.build(64, dev, torch.Generator().manual_seed(8))
    segs = [engine.Seg(engine.Act(t)) for t in x]
    n0 = nat.tc_launch_count()
    y_tc = L.forward(segs).t
    assert nat.tc_launch_count() == n0 + 1, 'tensor-core path not taken'
    d = L._fwd_desc(segs, 2, 32, 32)
    y_fp = torch.empty_like(y_tc)
    nat.check(lib.nlt_gconv_fwd(C.byref(d), nat.ptr(L.bias), nat.ACT_CODES['leakyrelu'], 0.0, None, 0, nat.ptr(y_fp),
                                nat.stream()))
    assert nat.tc_launch_count() == n0 + 1
    err = float((y_tc - y_fp).abs().max() / y_fp.abs().max())
    assert err <= 4e-6, err


def test_gconv_sub_and_bcast_segments():
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(0)
    N, H, W = 4, 8, 8
    a, b = torch.rand(N, H, W, 3), torch.rand(N, H, W, 3)
    ov = torch.randn(1, H, W, 8)
    q = torch.randn(N, H, W, 8)
    L = engine.ConvLayer('conv', 1, 1, 16)
    L.build(3, dev, torch.Generator().manual_seed(2))
    bg = b.to(dev)
    y = L.forward([engine.Seg(engine.Act(a.to(dev)), sub=bg)])
    _close(y.t, O.conv2d_same((a - b).double(), L.kernel.double().cpu(), L.bias.double().cpu(), 1))
    L1 = engine.ConvLayer('conv', 1, 1, 12, 'leakyrelu')          # pointwise kernel with a broadcast source
    L1.build(16, dev, torch.Generator().manual_seed(4))
    y = L1.forward([engine.Seg(engine.Act(q.to(dev))), engine.Seg(engine.Act(ov.to(dev)), bcast=True)])
    x = torch.cat((q, ov.expand(N, -1, -1, -1)), 3).double()
    _close(y.t, O.act(O.conv2d_same(x, L1.kernel.double().cpu(), L1.bias.double().cpu(), 1), 'leakyrelu'))
    L2 = engine.ConvLayer('conv', 2, 2, 16, 'relu')
    L2.build(16, dev, torch.Generator().manual_seed(3))
    y = L2.forward([engine.Seg(engine.Act(q.to(dev))), engine.Seg(engine.Act(ov.to(dev)), bcast=True)])
    x = torch.cat((q, ov.expand(N, -1, -1, -1)), 3).double()
    _close(y.t, O.act(O.conv2d_same(x, L2.kernel.double().cpu(), L2.bias.double().cpu(), 2), 'relu'))


def test_gconv_accumulates_two_consumers_and_elu():
    """One tensor feeding two convs: the second dgrad accumulates (beta=1) and
    applies the ELU derivative mask once, as the last contributor."""
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(4)
    x = torch.randn(2, 8, 8, 8)
    L0 = engine.ConvLayer('conv', 1, 1, 16, 'elu'); L0.build(8, dev, torch.Generator().manual_seed(5))
    L1 = engine.ConvLayer('conv', 2, 2, 8, None); L1.build(16, dev, torch.Generator().manual_seed(6))
    L2 = engine.ConvLayer('deconv', 2, 1, 4, None); L2.build(16, dev, torch.Generator().manual_seed(7))
    tape = engine.Tape()
    h = L0.forward([engine.Seg(engine.Act(x.to(dev)))], tape)
    y1 = L1.forward([engine.Seg(h)], tape)
    y2 = L2.forward([engine.Seg(h)], tape)
    p = {n: getattr(L, n).double().cpu().requires_grad_(True) for L in (L0,) for n in ('kernel', 'bias')}
    h64 = O.act(O.conv2d_same(x.double(), p['kernel'], p['bias'], 1), 'elu')
    y164 = O.conv2d_same(h64, L1.kernel.double().cpu(), L1.bias.double().cpu(), 2)
    y264 = O.conv2d_transpose_same(h64, L2.kernel.double().cpu(), L2.bias.double().cpu(), 1)
    g1, g2 = torch.randn_like(y164), torch.randn_like(y264)
    ((y164 * g1).sum() + (y264 * g2).sum()).backward()
    y1.grad, y2.grad = g1.float().to(dev), g2.float().to(dev)
    tape.backward()
    _close(L0.gkernel, p['kernel'].grad, rtol=1e-4, atol=1e-4)
    _close(L0.gbias, p['bias'].grad, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('K,B', [(2, 3), (6, 2)])
def test_kmean(K, B):
    engine, nat = _mods()
    dev = torch.device('cuda')
    torch.manual_seed(K)
    x = torch.randn(K * B, 4, 4, 8)
    a = engine.Act(x.to(dev), act='leakyrelu', needs_grad=True)
    tape = engine.Tape()
    m = engine.kmean(a, K, tape)
    want = x.view(K, B, 4, 4, 8).mean(0)
    _close(m.t, want)
    g = torch.randn(B, 4, 4, 8)
    m.grad = g.to(dev)
    tape.backward()
    want_g = (g / K).repeat(K, 1, 1, 1) * torch.where(x > 0, 1.0, 0.3)
    _close(a.grad, want_g)


@pytest.mark.parametrize('H,ih', [(16, 16), (32, 24)])
def test_uv2cam_forward_backward(H, ih):
    engine, nat = _mods()
    from util import synth
    dev = torch.device('cuda')
    lib = nat.lib()
    B = 2
    bt = synth.make_batch(B, H, ih, seed=11)
    base, warp, rgb_c = bt[1], bt[4], bt[6]
    # add edge / out-of-range sample points
    warp = warp.clone()
    warp[0, 0, :6] = torch.tensor([[-0.01, 0.5], [1.0, 0.5], [0.999, 0.999], [0.5, -0.2], [0.0, 0.0], [1.02, 0.3]])
    net_out = torch.randn(B, H, H, 3)
    out = {k: torch.empty(B, ih, ih, 3, device=dev) for k in ('pred', 'base', 'fg', 'gt')}
    pred_uv = torch.empty(B, H, H, 3, device=dev)
    # keep the device copies alive: the library only sees raw pointers
    g_net, g_base, g_warp, g_rgb = (t.to(dev).contiguous() for t in (net_out, base, warp, rgb_c))
    nat.check(lib.nlt_uv2cam_fwd(nat.ptr(g_net), nat.ptr(g_base), nat.ptr(g_warp), nat.ptr(g_rgb), B, H, H,
                                 ih, ih, 1, nat.ptr(pred_uv), nat.ptr(out['pred']), nat.ptr(out['base']),
                                 nat.ptr(out['fg']), nat.ptr(out['gt']), nat.stream()))
    n64 = net_out.double().requires_grad_(True)
    pred = O.set_left_top_corner(n64 + base.double(), 0)
    w = torch.stack((warp[..., 0].double() * H, warp[..., 1].double() * H), 3)
    # the kernel multiplies warp*uvw in fp32 like the reference; feed the oracle the same fp32 products
    w = torch.stack((warp[..., 0] * H, warp[..., 1] * H), 3).double()
    pc = O.resampler(pred, w)
    fg = O.resampler(O.set_left_top_corner(torch.ones_like(pred), 0), w)
    bc = O.resampler(O.set_left_top_corner(base.double(), 0), w)
    _close(pred_uv, pred, atol=1e-6)
    _close(out['pred'], pc, atol=2e-6)
    _close(out['base'], bc, atol=2e-6)
    _close(out['fg'], fg, atol=2e-6)
    _close(out['gt'], rgb_c.double() * fg, atol=2e-6)
    g = torch.randn(B, ih, ih, 3)
    pc.backward(g.double())
    dn = torch.empty(B, H, H, 3, device=dev)
    g_g = g.to(dev).contiguous()
    nat.check(lib.nlt_uv2cam_bwd(nat.ptr(g_g), nat.ptr(g_warp), B, H, H, ih, ih, nat.ptr(dn), nat.stream()))
    torch.cuda.synchronize()
    _close(dn, n64.grad, rtol=1e-4, atol=1e-5)
    assert float(dn[:, 0, 0].abs().max()) == 0.0


@pytest.mark.parametrize('shape,new', [((8, 8), (16, 16)), ((12, 10), (5, 7))])
def test_resize(shape, new):
    engine, nat = _mods()
    dev = torch.device('cuda')
    lib = nat.lib()
    x = torch.randn(2, shape[0], shape[1], 3)
    y = torch.empty(2, new[0], new[1], 3, device=dev)
    xg = x.to(dev)
    nat.check(lib.nlt_resize_bilinear_fwd(nat.ptr(xg), 2, shape[0], shape[1], 3, new[0], new[1], nat.ptr(y),
                                          nat.stream()))
    x64 = x.double().requires_grad_(True)
    y64 = O.resize_bilinear(x64, *new)
    _close(y, y64, atol=1e-6)
    g = torch.randn(2, new[0], new[1], 3)
    y64.backward(g.double())
    dx = torch.empty_like(x, device=dev)
    gg = g.to(dev)
    nat.check(lib.nlt_resize_bilinear_bwd(nat.ptr(gg), 2, shape[0], shape[1], 3, new[0], new[1], nat.ptr(dx),
                                          nat.stream()))
    _close(dx, x64.grad, atol=1e-5)


@pytest.mark.parametrize('hw', [(20, 24), (5, 7), (256, 192)])      # float4 path / scalar path (105 floats per sample) / many blocks
def test_l2_loss_and_grad(hw):
    import losses
    dev = torch.device('cuda')
    torch.manual_seed(1)
    pred, gt = torch.rand(3, hw[0], hw[1], 3), torch.rand(3, hw[0], hw[1], 3)
    L = losses.L2()
    L.grad_scale = 0.25
    got = L(gt.to(dev), pred.to(dev), keep_batch=True)
    p64 = pred.double().requires_grad_(True)
    want = O.l2_loss(gt.double(), p64, keep_batch=True)
    _close(got, want, rtol=1e-5, atol=1e-7)
    (want.sum() * 0.25).backward()
    _close(L.d_pred, p64.grad, rtol=1e-5, atol=1e-8)
    L.grad_scale = None
    got = L(gt.to(dev), pred.to(dev))
    _close(got, O.l2_loss(gt.double(), pred.double()), rtol=1e-5, atol=1e-7)


def test_amsgrad_kernel():
    engine, nat = _mods()
    dev = torch.device('cuda')
    lib = nat.lib()
    torch.manual_seed(2)
    n = 1000
    p = torch.randn(n); m = torch.zeros(n); v = torch.zeros(n); vh = torch.zeros(n)
    pg, mg, vg, vhg = (t.clone().to(dev) for t in (p, m, v, vh))
    p64, m64, v64, vh64 = (t.double() for t in (p, m, v, vh))
    for t in range(1, 5):
        g = torch.randn(n) * (0.5 if t != 3 else 0.01)
        gg = g.to(dev)
        nat.check(lib.nlt_amsgrad_step(nat.ptr(pg), nat.ptr(gg), nat.ptr(mg), nat.ptr(vg), nat.ptr(vhg), n, t,
                                       1e-3, 0.9, 0.999, 1e-7, 1.0, nat.stream()))
        p64, m64, v64, vh64 = O.amsgrad_step(p64, g.double(), m64, v64, vh64, t, 1e-3)
    # (1 - beta) is formed in fp32 (as TF's fp32 kernel does): 1 - 0.999f differs from 1e-3 by 4.7e-5 relative
    _close(pg, p64, rtol=1e-5, atol=2e-6)
    _close(vhg, vh64, rtol=2e-4, atol=1e-9)


def test_bad_arguments_raise():
    engine, nat = _mods()
    lib = nat.lib()
    d = nat.GConvDesc()
    rc = lib.nlt_gconv_fwd(C.byref(d), None, 0, 0.0, None, 0, None, None)
    assert rc == -1 and b'geometry' in lib.nlt_last_error()
    with pytest.raises(nat.NativeError):
        nat.ptr(torch.zeros(4))            # CPU tensor: no CPU fallback
    with pytest.raises(nat.NativeError):
        nat.ptr(torch.zeros(4, 4, device='cuda').t())
