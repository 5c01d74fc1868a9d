"""Tensor-core (mma.sync, 3xTF32) form of the depth-to-space input gradient of the 2x2 / stride-2 convs
(pwd2s_mma_kernel, option pwmma): same oracle checks as the FMA kernel it replaces, on every (K, CS) pair, with
lattice rows narrower than, equal to and wider than a tile; the FMA kernel must still run with pwmma = 0 or tc = 0."""
import pytest
import torch

from tests.test_gpu_ops import test_final_conv_input_gradient_rides_on_down_conv_dgrad as fused_check
from tests.test_gpu_ops import test_gconv_forward_backward as oracle_check

pytestmark = pytest.mark.gpu

# (H, W, sources, cout) of a 2x2 / stride-2 conv: its input gradient has K = cout channels into CS = source channels.
# Tiles are 128 lattice pixels (CS = 16) or 64 (CS = 32); the lattice width is W / 2.
D2S_SHAPES = [
    (16, 64, [16], 16),          # K 16, CS 16: rows of 32 < tile
    (4, 256, [16], 16),          # ... rows of 128 = tile
    (2, 1024, [16, 16], 16),     # ... rows of 512 > tile, two sources
    (16, 64, [16], 32),          # K 32, CS 16
    (4, 256, [16, 16], 32),
    (2, 1024, [16], 32),
    (16, 32, [32], 32),          # K 32, CS 32: rows of 16 < tile
    (4, 128, [32], 32),          # ... rows of 64 = tile
    (2, 512, [32, 32], 32),      # ... rows of 256 > tile
]


@pytest.mark.parametrize('H,W,segc,cout', D2S_SHAPES)
@pytest.mark.parametrize('act', ['leakyrelu', None])
def test_pwd2s_mma_input_gradient(H, W, segc, cout, act):
    import nlt_native as nat
    for opts, kernel in (({'pwmma': 1, 'tc': 1}, 'pwd2s_mma_kernel'), ({'pwmma': 0, 'tc': 1}, 'pwd2s_kernel'),
                         ({'pwmma': 1, 'tc': 0}, 'pwd2s_kernel')):
        with nat.options(**opts):
            n0 = nat.kernel_launch_count(kernel)
            oracle_check('conv', 2, 2, H, W, segc, cout, act)
            assert nat.kernel_launch_count(kernel) > n0, '%s did not run with %s' % (kernel, opts)


# (H, W, c_skip, c_other, down_cout, dk): the fused pointwise term (fused arm) and beta = 1 (unfused arm: the down-conv's
# input gradient adds to the final conv's) on the new kernel
@pytest.mark.parametrize('H,W,c_skip,c_other,down_cout,dk', [
    (8, 512, 16, 4, 16, 2), (4, 1024, 16, 4, 32, 2), (4, 512, 32, 4, 32, 2)])
def test_pwd2s_mma_fused_term_and_beta(H, W, c_skip, c_other, down_cout, dk):
    import nlt_native as nat
    with nat.options(pwmma=1, tc=1):
        n0 = nat.kernel_launch_count('pwd2s_mma_kernel')
        fused_check(H, W, c_skip, c_other, down_cout, dk)
        assert nat.kernel_launch_count('pwd2s_mma_kernel') >= n0 + 2, 'pwd2s_mma_kernel did not run on both arms'


def test_pwd2s_mma_graph_replay_matches_eager():
    """A layer's forward + backward captured in a CUDA graph gives the same bits as the eager launches."""
    import engine
    import nlt_native as nat
    dev = torch.device('cuda')
    torch.manual_seed(3)
    with nat.options(pwmma=1, tc=1):
        side_streams = engine.USE_SIDE_STREAM
        engine.USE_SIDE_STREAM = False          # weight gradients on the capturing stream (no fork / join in this graph)
        try:
            L = engine.ConvLayer('conv', 2, 2, 32, 'leakyrelu')
            L.build(32, dev, torch.Generator().manual_seed(1))
            xs = [torch.randn(2, 8, 1024, 16, device=dev) for _ in range(2)]
            dz = torch.randn(2, 4, 512, 32, device=dev)
            grads = []

            def body():
                acts = [engine.Act(x, act='leakyrelu', needs_grad=True) for x in xs]
                tape = engine.Tape()
                y = L.forward([engine.Seg(a) for a in acts], tape)
                y.grad = dz.clone()
                tape.backward()
                grads[:] = [a.grad for a in acts]

            n0 = nat.kernel_launch_count('pwd2s_mma_kernel')
            ws = (engine.Workspace(), engine.Workspace())
            with engine.use_workspaces(*ws):
                body()
                torch.cuda.synchronize()
                eager = [g.clone() for g in grads]
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    body()
                torch.cuda.current_stream().wait_stream(side)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    body()
            assert nat.kernel_launch_count('pwd2s_mma_kernel') > n0
            for out in grads:
                out.fill_(float('nan'))
            g.replay()
            torch.cuda.synchronize()
            for a, b in zip(grads, eager):
                assert torch.equal(a, b)
            del g
        finally:
            engine.USE_SIDE_STREAM = side_streams
