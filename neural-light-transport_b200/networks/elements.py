"""Element factories with the reference's names (nlt/networks/elements.py:26-125).

Each factory returns a *spec* consumed by Block (networks/convnet.py); the
conv + norm + act triple of the reference is executed as ONE fused CUDA op
(bias and activation live in the conv epilogue), so `norm`/`act`/`iden`
return markers rather than callable layers.
"""
from engine import ConvLayer, NormLayer, PoolLayer  # noqa: F401


def conv(kernel_size, n_ch_out, stride=1):
    return ConvLayer('conv', kernel_size, stride, n_ch_out)


def deconv(kernel_size, n_ch_out, stride=1):
    return ConvLayer('deconv', kernel_size, stride, n_ch_out)


def upconv(n_ch_out):
    """The conv half of `upconv` (UpSampling2D(2, 'bilinear') + Conv2D(n, 2, padding='same'), linear with bias).  The
    upsampling is done by the Block that owns it (networks/convnet.py), once per distinct source of its input."""
    return ConvLayer('conv', 2, 1, n_ch_out)


def norm(type_):
    """None -> identity; 'pixel' / 'instance' -> the kind of engine.NormLayer a block inserts between each conv and
    its activation.  'batch' couples the samples of a batch (the data-parallel split would change its statistics) and
    'layer' is unshipped: both stay NotImplementedError."""
    if type_ is None or type_.lower() == 'none':
        return None
    if type_ in ('pixel', 'instance'):
        return type_
    if type_ in ('batch', 'layer'):
        raise NotImplementedError('norm=%s is not on the accelerated path' % type_)
    raise NotImplementedError(type_)


def act(type_):
    if type_ in ('relu', 'leakyrelu', 'elu'):
        return type_
    raise NotImplementedError(type_)


def pool(type_):
    if type_ is None or type_.lower() == 'none':
        return None
    if type_ in ('max', 'avg'):
        return PoolLayer(type_)
    raise NotImplementedError(type_)


def iden():
    return None
