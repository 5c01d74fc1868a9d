"""UV-space encoder/decoder: the layer list behind `networks.convnet.Network` (interface of
nlt/networks/convnet.py:30-90).  Every entry of `.layers` is a callable `Block` (x -> y on NHWC CUDA tensors, or
on engine segments), which is what `nlt_test.extract_feat` and the two-stream walk of `models.nlt` iterate over.
"""
import numpy as np
import torch

from engine import Act, Seg, upsample2x
from util import net as netutil
from .seq import Network as BaseNetwork
from .elements import conv, norm, act, pool, deconv, upconv, NormLayer


class Block:
    """One entry of Network.layers: 1x1 conv, down block or up block, run as fused conv(+bias+act) CUDA ops; with
    `norm != None` every conv of a two-conv block is followed by an engine.NormLayer that carries the activation
    (conv -> norm -> act, nlt/networks/convnet.py:50-59, 67-76).  With `pool != None` a down block ends in an
    engine.PoolLayer and an up block starts with `upconv`: bilinear x2 of every distinct source of its input concat,
    then convs[0], a linear 2x2 conv (convnet.py:58, 67)."""

    def __init__(self, convs, norms=None, pool=None, upconv=False):
        self.convs = convs
        self.norms = norms if norms is not None else [None] * len(convs)
        self.pool = pool
        self.upconv = upconv

    @property
    def built(self):
        return all(c.built for c in self.convs)

    def param_layers(self):
        """[(suffix, layer)] of everything in this block that owns parameters, in registration order."""
        out = []
        for ci, (c, nm) in enumerate(zip(self.convs, self.norms)):
            out.append(('%d' % ci, c))
            if nm is not None and nm.has_params:
                out.append(('%d.norm' % ci, nm))
        return out

    def build(self, cin, device, generator=None):
        for c, nm in zip(self.convs, self.norms):
            if not c.built:
                c.build(cin, device, generator)
            cin = c.cout
            if nm is not None and not nm.built:
                nm.build(cin, device, generator)
        return cin

    def forward_segs(self, segs, tape=None):
        """segs: list of engine.Seg (virtual concat) -> engine.Act"""
        if self.upconv:
            segs = self._upsample(segs, tape)
        y = None
        for i, (c, nm) in enumerate(zip(self.convs, self.norms)):
            y = c.forward(segs if i == 0 else [Seg(y)], tape)
            if nm is not None:
                y = nm.forward(y, tape)
        if self.pool is not None:
            y = self.pool.forward(y, tape)
        return y

    @staticmethod
    def _upsample(segs, tape):
        """Each distinct source Act is upsampled once: the first up block reads [q, agg, q, agg] (the bottleneck
        concatenated with itself), which costs two upsamples, and the conv reads each result twice."""
        done = {}
        out = []
        for sg in segs:
            if sg.sub is not None:
                raise ValueError('upconv: a segment with a subtrahend cannot be upsampled')
            if id(sg.a) not in done:
                done[id(sg.a)] = upsample2x(sg.a, tape)
            out.append(Seg(done[id(sg.a)], bcast=sg.bcast))
        return out

    def __call__(self, x):
        if isinstance(x, Act):
            return self.forward_segs([Seg(x)])
        return self.forward_segs([Seg(Act(x.contiguous()))]).t


def _block_kinds(n_feat):
    """('down' | 'up', channels) for every entry of the channel schedule but the last: a block contracts when its
    channel count does not drop below the previous block's -- so 256 -> 256 is still a *down* block
    (nlt/networks/convnet.py:49), which is why depth 256 gives six downs and six ups."""
    kinds, prev = [], 0
    for n in n_feat[:-1]:
        kinds.append(('down' if n >= prev else 'up', n))
        prev = n
    return kinds


class Network(BaseNetwork):
    """Constructor signature, `.layers`, `.is_contracting` and `.spatsize_changes` of nlt/networks/convnet.py:30-90:
    [1x1 conv -> depth0] + one two-conv block per schedule entry (strided conv + conv when contracting, strided
    transposed conv + transposed conv when expanding, each followed by the activation) + [1x1 conv -> 3].
    `pool_type = max | avg` gives the classic U-Net: every down block ends in a 2x2 pool and every up block starts with
    `upconv(n)`.  Only `stride = 1` is accepted with a pool: at stride 2 each level shrinks by 4, and six levels would
    need UV sizes that are multiples of 4**6 for the reference's own skip concat (nlt/models/nlt.py:190)."""

    def __init__(self, depth0, depth, kernel, stride, norm_type=None, act_type='relu', pool_type=None):
        super().__init__()
        # unsupported normalisation / pooling kinds raise NotImplementedError right here, like the reference's
        # element factories; the supported kind for both is None (identity)
        norm_kind = norm(self.str2none(norm_type))
        pool_kind = pool(self.str2none(pool_type))
        activation = act(act_type)
        if pool_kind is not None and stride != 1:
            raise NotImplementedError(
                'pool=%s with stride=%d: every level would shrink the UV map by %d, so six levels need sizes that are '
                'multiples of %d**6; pooling networks take stride=1' % (pool_type, stride, 2 * stride, 2 * stride))
        n_feat = netutil.gen_feat_n(depth0, depth)

        def add(convs, contracting, scale, norms=None, **kw):
            self.layers.append(Block(convs, norms, **kw))
            self.is_contracting.append(contracting)
            self.spatsize_changes.append(scale)

        def pair(make, n):
            first, second = make(kernel, n, stride=stride), make(kernel, n, stride=1)
            if norm_kind is None:
                first.act = second.act = activation
                return [first, second], None
            # conv -> norm -> act: the activation moves into the norm op
            return [first, second], [NormLayer(norm_kind, activation), NormLayer(norm_kind, activation)]

        self.is_contracting, self.spatsize_changes = [], []
        add([conv(1, n_feat[0], stride=1)], True, 1)                 # full-resolution feature map
        for kind, n in _block_kinds(n_feat):
            if kind == 'down':
                convs, norms = pair(conv, n)
                if pool_kind is None:
                    add(convs, True, 1 / stride, norms)
                else:
                    add(convs, True, 1 / stride / 2, norms, pool=pool(self.str2none(pool_type)))
            else:
                convs, norms = pair(deconv, n)
                if pool_kind is None:
                    add(convs, False, stride, norms)
                else:
                    # [upconv conv, deconv, deconv]: param_layers() names them conv0 / conv1 / conv2
                    add([upconv(n)] + convs, False, stride * 2, None if norms is None else [None] + norms,
                        upconv=True)
        add([conv(1, n_feat[-1], stride=1)], False, 1)               # back to 3 channels
        assert float(np.prod(self.spatsize_changes)) == 1, "Resolution doesn't return to the original value"

    def conv_layers(self):
        return [c for blk in self.layers for c in blk.convs]

    def param_layers(self):
        return [layer for blk in self.layers for _, layer in blk.param_layers()]
