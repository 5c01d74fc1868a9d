"""CPU oracle of the LPIPS loss (nlt/losses.py:121-169).  TEST INFRASTRUCTURE ONLY.

The reference runs LPIPS as a frozen TensorFlow graph, `third_party/lpips/net-lin_alex_v0.1.pb`.  That file cannot be
shipped here; `fetch_graph()` (called by build()) copies it from a reference checkout into oracle/_ref/, which is
never committed, and checks its sha256.  Two restatements pin the CUDA loss:

  (a) run_graph      a float64 interpreter of the frozen GraphDef itself, op by op (the 27 op kinds the graph uses).
                     It pins the computation to the reference's own file rather than to a reading of it.
  (b) lpips_torch    the same computation written out in float64 torch with autograd, for gradients.  Its backward
                     can take given ReLU masks (the product's, so that a feature whose sign differs in the last bit
                     does not count as an error) and treats an all-zero pred feature vector as the CUDA kernels do:
                     the normalisation's gradient term is 0 there (the reference's TF gradient is NaN).
"""
import hashlib
import os
import shutil

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, 'oracle', '_ref')
GRAPH = os.path.join(REF_DIR, 'net-lin_alex_v0.1.pb')
# a reference checkout next to this repository, unless NLT_REFERENCE names one
REFERENCE = os.environ.get('NLT_REFERENCE', os.path.join(os.path.dirname(ROOT), 'reference'))
SHA256 = 'ef6658df105db18da7fb6c7dc067c59f853738f244dfab90176a8a22092f5227'


def _sha(path):
    with open(path, 'rb') as f:
        return hashlib.sha256(f.read()).hexdigest()


def fetch_graph():
    """Copies the reference's LPIPS graph into oracle/_ref/ (sha256-checked).  Without a reference checkout a verified
    copy that is already there is kept; returns its path, or None when there is neither."""
    src = os.path.join(REFERENCE, 'third_party', 'lpips', 'net-lin_alex_v0.1.pb')
    if os.path.isfile(GRAPH) and _sha(GRAPH) == SHA256:
        return GRAPH
    if not os.path.isfile(src):
        return None
    if _sha(src) != SHA256:
        raise ValueError('%s: sha256 differs from the LPIPS graph the kernels were checked against' % src)
    os.makedirs(REF_DIR, exist_ok=True)
    tmp = GRAPH + '.tmp'
    shutil.copyfile(src, tmp)
    os.replace(tmp, GRAPH)
    return GRAPH


def graph_path():
    """The verified copy in oracle/_ref/, or None."""
    return GRAPH if os.path.isfile(GRAPH) and _sha(GRAPH) == SHA256 else None


# ---------------------------------------------------------------------------------------------------------------------
# (a) the frozen graph, interpreted in float64
# ---------------------------------------------------------------------------------------------------------------------
def _conv2d_nhwc(x, w_hwio, strides, padding):
    assert padding == 'VALID'
    xt = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 3, 1, 2)))
    wt = torch.from_numpy(np.ascontiguousarray(w_hwio.transpose(3, 2, 0, 1)))
    y = torch.nn.functional.conv2d(xt, wt, stride=(strides[1], strides[2]))
    return y.numpy().transpose(0, 2, 3, 1)


def _maxpool_nhwc(x, ksize, strides, padding):
    assert padding == 'VALID'
    xt = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 3, 1, 2)))
    y = torch.nn.functional.max_pool2d(xt, (ksize[1], ksize[2]), (strides[1], strides[2]))
    return y.numpy().transpose(0, 2, 3, 1)


def run_graph(nodes, pred, gt, output='Reshape_10'):
    """Evaluates `output` of the parsed graph (util.tf_graphdef.parse_graph) on NCHW float64 inputs 0 = pred and
    1 = gt, both already mapped to [-1, 1] (nlt/losses.py:151-164).  Float constants are promoted to float64."""
    memo = {}

    def val(ref):
        name, _, k = ref.partition(':')
        out = ev(name)
        return out[int(k)] if k else (out[0] if isinstance(out, list) else out)

    def ev(name):
        if name in memo:
            return memo[name]
        n = nodes[name]
        a = [val(i) for i in n.inputs if not i.startswith('^')]
        at, op = n.attr, n.op
        if op == 'Const':
            v = at['value']
            r = v.astype(np.float64) if v.dtype.kind == 'f' else v
        elif op == 'Placeholder':
            r = {'0': pred, '1': gt}[name]
        elif op == 'Identity':
            r = a[0]
        elif op == 'Transpose':
            r = np.transpose(a[0], a[1])
        elif op == 'Pad':
            r = np.pad(a[0], a[1])
        elif op == 'Split':
            r = np.split(a[1], at['num_split'], axis=int(a[0]))
        elif op == 'ConcatV2':
            r = np.concatenate(a[:-1], axis=int(a[-1]))
        elif op == 'Conv2D':
            assert at.get('data_format', 'NHWC') == 'NHWC' and list(at.get('dilations', [1] * 4)) == [1] * 4
            r = _conv2d_nhwc(a[0], a[1], at['strides'], at['padding'])
        elif op == 'MaxPool':
            assert at.get('data_format', 'NHWC') == 'NHWC'
            r = _maxpool_nhwc(a[0], at['ksize'], at['strides'], at['padding'])
        elif op == 'Relu':
            r = np.maximum(a[0], 0)
        elif op in ('Add', 'Sub', 'RealDiv', 'Pow', 'Equal'):
            r = {'Add': np.add, 'Sub': np.subtract, 'RealDiv': np.divide, 'Pow': np.power,
                 'Equal': np.equal}[op](a[0], a[1])
        elif op == 'Sqrt':
            r = np.sqrt(a[0])
        elif op in ('Sum', 'Mean'):
            r = (np.sum if op == 'Sum' else np.mean)(a[0], axis=tuple(np.atleast_1d(a[1]).tolist()),
                                                     keepdims=bool(at.get('keep_dims', False)))
        elif op == 'Reshape':
            r = np.reshape(a[0], a[1])
        elif op == 'Shape':
            r = np.array(np.shape(a[0]), dtype=np.int64 if at.get('out_type') == 9 else np.int32)
        elif op == 'Slice':
            begin, size = a[1], a[2]
            r = a[0][tuple(slice(b, None if s == -1 else b + s) for b, s in zip(begin, size))]
        elif op == 'Squeeze':
            dims = at.get('squeeze_dims') or [i for i, d in enumerate(np.shape(a[0])) if d == 1]
            r = np.squeeze(a[0], axis=tuple(d % max(np.ndim(a[0]), 1) for d in dims))
        elif op == 'ExpandDims':
            r = np.expand_dims(a[0], int(a[1]))
        elif op == 'Where':
            r = np.argwhere(a[0]).astype(np.int64)
        elif op == 'GatherV2':
            r = np.take(a[0], a[1], axis=int(a[2]))
        elif op == 'Cast':
            r = np.asarray(a[0]).astype({1: np.float32, 2: np.float64, 3: np.int32, 9: np.int64}[at['DstT']])
        elif op == 'SparseToDense':
            idx, shape, values, default = a
            shape = np.asarray(shape).reshape(-1)
            r = np.full(shape, default, dtype=np.asarray(values).dtype)
            idx = np.asarray(idx).reshape(-1, len(shape))
            for row, v in zip(idx, np.broadcast_to(values, (len(idx),))):
                r[tuple(row)] = v
        else:
            raise NotImplementedError('graph op %s (%s)' % (op, name))
        memo[name] = r
        return r

    return val(output)


def graph_lpips(nodes, pred, gt):
    """Per-sample LPIPS of NHWC images in [0, 1] by the graph interpreter: float64 [N]."""
    def prep(v):
        return np.ascontiguousarray((np.asarray(v, dtype=np.float64) * 2 - 1).transpose(0, 3, 1, 2))
    return run_graph(nodes, prep(pred), prep(gt)).reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------
# (b) torch float64 restatement with autograd
# ---------------------------------------------------------------------------------------------------------------------
class _MaskedRelu(torch.autograd.Function):
    """ReLU whose backward uses the given mask (1 where the product's feature is > 0) instead of its own sign."""

    @staticmethod
    def forward(ctx, x, mask):
        ctx.save_for_backward(mask if mask is not None else (x > 0))
        return torch.relu(x)

    @staticmethod
    def backward(ctx, g):
        (m,) = ctx.saved_tensors
        return g * m.to(g.dtype), None


def _norm(f):
    """|f| over channels (dim 1) with d|f|/df taken as 0 where |f| = 0 (the clamp's gradient is 0 below the smallest
    normal number, whose square root leaves |f| + 1e-10 unchanged)."""
    return torch.sqrt((f * f).sum(1, keepdim=True).clamp_min(torch.finfo(f.dtype).tiny))


def features(weights, x, masks=None):
    """The five ReLU outputs of AlexNet on NCHW x (already scaled; float64, or float32 for an emulation of the fp32
    reference); masks: optional list of five NCHW bool tensors for the backward pass."""
    w = {k: torch.as_tensor(v, dtype=x.dtype, device=x.device) for k, v in weights.items()}
    feats = []
    pads, strides = (2, 2, 1, 1, 1), (4, 1, 1, 1, 1)
    for i in range(5):
        if i in (1, 2):
            x = torch.nn.functional.max_pool2d(x, 3, 2)
        x = torch.nn.functional.conv2d(x, w['w%d' % (i + 1)], w['b%d' % (i + 1)], stride=strides[i], padding=pads[i])
        x = _MaskedRelu.apply(x, None if masks is None else masks[i])
        feats.append(x)
    return feats


def lpips_torch(weights, pred, gt, masks=None):
    """Per-sample LPIPS [N] of NHWC images in [0, 1] (float64 tensors, or float32 for an emulation of the fp32
    reference; pred may require grad).  masks: optional five NHWC bool tensors of the pred half's ReLU outputs, used by
    the backward pass of the pred branch."""
    w = {k: torch.as_tensor(v, dtype=pred.dtype, device=pred.device) for k, v in weights.items()}

    def prep(v):
        x = (v * 2 - 1).permute(0, 3, 1, 2)
        return x * w['scale'].view(1, 3, 1, 1) + w['shift'].view(1, 3, 1, 1)
    mk = None if masks is None else [m.permute(0, 3, 1, 2) for m in masks]
    fp = features(weights, prep(pred), mk)
    fg = features(weights, prep(gt))
    total = 0
    for i in range(5):
        up = fp[i] / (_norm(fp[i]) + 1e-10)
        ug = fg[i] / (_norm(fg[i]) + 1e-10)
        d = ((up - ug) ** 2 * w['lin%d' % (i + 1)].view(1, -1, 1, 1)).sum(1)
        total = total + d.mean((1, 2))
    return total



def relu_masks(weights, pred):
    """The five ReLU masks (NHWC bool) of the pred branch of a float64 forward (for counting flipped masks)."""
    w = {k: torch.as_tensor(v, dtype=torch.float64, device=pred.device) for k, v in weights.items()}
    x = (pred * 2 - 1).permute(0, 3, 1, 2) * w['scale'].view(1, 3, 1, 1) + w['shift'].view(1, 3, 1, 1)
    with torch.no_grad():
        return [f.permute(0, 2, 3, 1) > 0 for f in features(weights, x)]
