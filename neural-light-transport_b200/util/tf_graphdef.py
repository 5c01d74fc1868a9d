"""Reader of TensorFlow GraphDef files (frozen graphs), and of the one frozen graph the reference's LPIPS loss runs:
`third_party/lpips/net-lin_alex_v0.1.pb`, loaded by nlt/losses.py:143-169.  The protobuf wire decoder is the one of
util/tf_ckpt.py.

Messages read (tensorflow/core/framework/*.proto, public):
  GraphDef    node = 1 (NodeDef)
  NodeDef     name = 1, op = 2, input = 3 ("name" or "name:k"; "^name" is a control input), attr = 5 (map<string,
              AttrValue>: key = 1, value = 2)
  AttrValue   list = 1 (ListValue: s = 2, i = 3, f = 4, type = 6), s = 2, i = 3, f = 4, b = 5, type = 6, shape = 7,
              tensor = 8
  TensorProto dtype = 1, tensor_shape = 2 (dim = 2 {size = 1}), tensor_content = 4, float_val = 5, double_val = 6,
              int_val = 7, bool_val = 11, int64_val = 10
"""
import struct

import numpy as np

from util.tf_ckpt import _DTYPES, _parse_fields, _varint

LPIPS_ALEX_SHA256 = 'ef6658df105db18da7fb6c7dc067c59f853738f244dfab90176a8a22092f5227'


class Node():
    def __init__(self, name, op, inputs, attr):
        self.name, self.op, self.inputs, self.attr = name, op, inputs, attr

    def __repr__(self):
        return 'Node(%s %s <- %s)' % (self.name, self.op, self.inputs)


def _packed(v, wt, fmt):
    """Values of a repeated scalar field: one element (wire type 0/1/5) or a packed run (wire type 2)."""
    if wt != 2:
        return [struct.unpack('<' + fmt, struct.pack('<' + {'f': 'I', 'd': 'Q'}[fmt], v))[0]] if fmt in 'fd' else [v]
    if fmt in 'fd':
        return list(struct.unpack('<%d%s' % (len(v) // struct.calcsize(fmt), fmt), v))
    out, pos = [], 0
    while pos < len(v):
        x, pos = _varint(v, pos)
        out.append(x)
    return out


def _signed(x):
    return x - (1 << 64) if x >= 1 << 63 else x


def _shape(buf):
    dims = []
    for num, _, v in _parse_fields(buf):
        if num == 2:
            size = 0
            for n2, _, v2 in _parse_fields(v):
                if n2 == 1:
                    size = _signed(v2)
            dims.append(size)
    return dims


def _tensor(buf):
    dtype, shape, content, vals = 0, [], None, []
    for num, wt, v in _parse_fields(buf):
        if num == 1:
            dtype = v
        elif num == 2:
            shape = _shape(v)
        elif num == 4:
            content = v
        elif num == 5:
            vals += _packed(v, wt, 'f')
        elif num == 6:
            vals += _packed(v, wt, 'd')
        elif num in (7, 10, 11):
            vals += [_signed(x) for x in _packed(v, wt, 'i')]
    if dtype not in _DTYPES:
        raise ValueError('unsupported tensor dtype %d' % dtype)
    dt = np.dtype(_DTYPES[dtype])
    n = int(np.prod(shape)) if shape else 1
    if content is not None:
        if len(content) != n * dt.itemsize:
            raise ValueError('tensor content of %d bytes for shape %s' % (len(content), shape))
        return np.frombuffer(content, dtype=dt.newbyteorder('<')).astype(dt).reshape(shape)
    if not vals:
        vals = [0]
    if len(vals) != n and len(vals) != 1:
        raise ValueError('%d tensor values for shape %s' % (len(vals), shape))
    return np.broadcast_to(np.array(vals, dtype=dt), (n,)).reshape(shape).copy()


def _attr(buf):
    f = {num: (wt, v) for num, wt, v in _parse_fields(buf)}
    if 1 in f:                                 # list
        out = []
        for num, wt, v in _parse_fields(f[1][1]):
            if num == 2:
                out.append(v.decode())
            elif num in (3, 6):
                out += [_signed(x) for x in _packed(v, wt, 'i')]
            elif num == 4:
                out += _packed(v, wt, 'f')
        return out
    if 2 in f:
        return f[2][1].decode()
    if 3 in f or 6 in f:
        return _signed(f.get(3, f.get(6))[1])
    if 4 in f:
        return _packed(f[4][1], f[4][0], 'f')[0]
    if 5 in f:
        return bool(f[5][1])
    if 7 in f:
        return _shape(f[7][1])
    if 8 in f:
        return _tensor(f[8][1])
    return None


def parse_graph(buf):
    """{node name: Node} of a serialized GraphDef; Const nodes carry their value as attr['value'] (ndarray)."""
    nodes = {}
    try:
        fields = _parse_fields(buf)
    except (IndexError, struct.error) as e:
        raise ValueError('not a GraphDef (truncated protobuf: %s)' % e)
    for num, _, v in fields:
        if num != 1:
            continue
        name, op, inputs, attr = '', '', [], {}
        try:
            for n2, _, v2 in _parse_fields(v):
                if n2 == 1:
                    name = v2.decode()
                elif n2 == 2:
                    op = v2.decode()
                elif n2 == 3:
                    inputs.append(v2.decode())
                elif n2 == 5:
                    kv = {n3: v3 for n3, _, v3 in _parse_fields(v2)}
                    attr[kv[1].decode()] = _attr(kv.get(2, b''))
        except (IndexError, KeyError, struct.error, UnicodeDecodeError) as e:
            raise ValueError('not a GraphDef (corrupt node: %s)' % e)
        nodes[name] = Node(name, op, inputs, attr)
    if not nodes:
        raise ValueError('not a GraphDef (no nodes)')
    return nodes


def load_graph(path):
    with open(path, 'rb') as f:
        return parse_graph(f.read())


# ---------------------------------------------------------------------------------------------------------------------
# The LPIPS AlexNet graph
# ---------------------------------------------------------------------------------------------------------------------
# conv: (Cout, Cin, k, stride, pad); a MaxPool 3x3 / s2 VALID follows the ReLU of conv1 and conv2
ALEX = ((64, 3, 11, 4, 2), (192, 64, 5, 1, 2), (384, 192, 3, 1, 1), (256, 384, 3, 1, 1), (256, 256, 3, 1, 1))
POOL_AFTER = (True, True, False, False, False)
NCHW_TO_NHWC, NHWC_TO_NCHW, OIHW_TO_HWIO = [0, 2, 3, 1], [0, 3, 1, 2], [2, 3, 1, 0]


class _Walk():
    def __init__(self, nodes):
        self.nodes = nodes

    def fail(self, msg):
        raise ValueError('not the LPIPS AlexNet graph: ' + msg)

    def get(self, ref, op=None):
        n = self.nodes.get(ref.split(':')[0])
        if n is None:
            self.fail('missing node %s' % ref)
        if op is not None and n.op != op:
            self.fail('%s is %s, expected %s' % (n.name, n.op, op))
        return n

    def inp(self, node, i, op=None):
        if len(node.inputs) <= i:
            self.fail('%s has %d inputs' % (node.name, len(node.inputs)))
        return self.get(node.inputs[i], op)

    def value(self, node, shape=None):
        v = node.attr.get('value') if node.op == 'Const' else None
        if not isinstance(v, np.ndarray) or (shape is not None and tuple(v.shape) != tuple(shape)):
            self.fail('%s: expected a constant of shape %s, got %s' % (node.name, shape, getattr(v, 'shape', node.op)))
        return v

    def transpose(self, node, perm):
        if node.op != 'Transpose' or list(self.value(self.inp(node, 1))) != perm:
            self.fail('%s: expected Transpose %s' % (node.name, perm))
        return self.inp(node, 0)

    def conv(self, conv, stride, wshape, groups=1, index=0):
        """Checks output `index` of Conv2D(Split(Transpose(Pad(x))), Split(Transpose(W))); returns (x, pad, W value)."""
        a = conv.attr
        if conv.op != 'Conv2D' or a.get('padding') != 'VALID' or a.get('data_format', 'NHWC') != 'NHWC' or \
                list(a.get('strides', [])) != [1, stride, stride, 1] or list(a.get('dilations', [1] * 4)) != [1] * 4:
            self.fail('%s: expected a VALID NHWC Conv2D of stride %d, got %s %s' % (
                conv.name, stride, conv.op, {k: a.get(k) for k in ('strides', 'padding', 'dilations')}))
        port = ':%d' % index if index else ''
        xs, ws = self.inp(conv, 0, 'Split'), self.inp(conv, 1, 'Split')
        if conv.inputs[0] != xs.name + port or conv.inputs[1] != ws.name + port or \
                xs.attr.get('num_split') != groups or ws.attr.get('num_split') != groups:
            self.fail('%s: expected group %d of %d' % (conv.name, index, groups))
        pad = self.transpose(self.inp(xs, 1), NCHW_TO_NHWC)
        if pad.op != 'Pad':
            self.fail('%s: expected Pad, got %s' % (pad.name, pad.op))
        pc = self.value(self.inp(pad, 1), (4, 2))
        p = int(pc[2, 0])
        if (pc[:2] != 0).any() or (pc[2:] != p).any():
            self.fail('%s: pad %s is not symmetric spatial padding' % (pad.name, pc.tolist()))
        w = self.value(self.transpose(self.inp(ws, 1), OIHW_TO_HWIO), wshape)
        return self.inp(pad, 0), p, w

    def kernel_shape(self, conv):
        """Shape of the constant behind a Conv2D's kernel operand, None when it is not Split(Transpose(Const))."""
        try:
            return tuple(self.value(self.inp(self.inp(self.inp(conv, 1, 'Split'), 1, 'Transpose'), 0)).shape)
        except ValueError:
            return None

    def layer(self, relu):
        """Relu(Transpose(Add(Identity(Conv2D), bias))) -> (conv node, bias value)."""
        add = self.transpose(self.inp(relu, 0), NHWC_TO_NCHW)
        if add.op != 'Add':
            self.fail('%s: expected Add, got %s' % (add.name, add.op))
        conv = self.inp(add, 0)
        if conv.op == 'Identity':
            conv = self.inp(conv, 0)
        return conv, self.value(self.inp(add, 1))


def _keep(out, g, name, v):
    if name in out and not np.array_equal(out[name], v):
        g.fail('the pred and gt branches use different %s constants' % name)
    out[name] = v


def load_lpips_alex(path):
    """The 17 float32 constants of the frozen LPIPS AlexNet graph:
      scale [3], shift [3]          the scaling layer  x * scale + shift  (= (x - LPIPS shift) / LPIPS scale)
      w1 .. w5  [Cout, Cin, k, k]   conv kernels, OIHW as stored      b1 .. b5 [Cout]  biases
      lin1 .. lin5 [C]              the non-negative channel weights of the distance head
    Raises FileNotFoundError when the file is missing and ValueError when the graph is not the one the CUDA kernels
    implement (op kinds, strides, kernel sizes, padding, pad constants, shapes, or the two branches not sharing their
    constants)."""
    g = _Walk(load_graph(path))
    out, feats = {}, {}
    relus = [n for n in g.nodes.values() if n.op == 'Relu']
    for branch, placeholder in ((0, '0'), (1, '1')):
        feats[branch], prev = [], None
        for li, (co, ci, k, s, p) in enumerate(ALEX):
            hit = None
            for r in relus:
                conv, bias = g.layer(r)
                if g.kernel_shape(conv) != (co, ci, k, k):
                    continue
                src, pad, w = g.conv(conv, s, (co, ci, k, k))
                if li == 0:
                    src = g.transpose(src, NHWC_TO_NCHW)
                    if src.op != 'Add' or g.inp(src, 0).op != 'ConcatV2':
                        continue
                    cat, x = g.inp(src, 0), None
                    for j in range(3):      # the scale constant [3, 1, 1, 1], split into three 1x1 groups
                        xj, pj, scale = g.conv(g.get(cat.inputs[j]), 1, (3, 1, 1, 1), groups=3, index=j)
                        if pj != 0 or cat.inputs[j] != g.get(cat.inputs[j]).name or (x is not None and xj is not x):
                            g.fail('%s: scaling layer is not a per-channel scale of one input' % cat.name)
                        x = xj
                    if x.name != placeholder:
                        continue
                    _keep(out, g, 'scale', scale.reshape(3))
                    _keep(out, g, 'shift', g.value(g.inp(src, 1), (3,)))
                elif POOL_AFTER[li - 1]:
                    mp = g.transpose(src, NHWC_TO_NCHW)
                    if mp.op != 'MaxPool' or g.transpose(g.inp(mp, 0), NCHW_TO_NHWC).name != prev:
                        continue
                    a = mp.attr
                    if list(a.get('ksize', [])) != [1, 3, 3, 1] or list(a.get('strides', [])) != [1, 2, 2, 1] or \
                            a.get('padding') != 'VALID' or a.get('data_format', 'NHWC') != 'NHWC':
                        g.fail('%s: expected MaxPool 3x3 / s2 VALID NHWC' % mp.name)
                elif src.name != prev:
                    continue
                if pad != p:
                    g.fail('%s: pad %d, expected %d' % (conv.name, pad, p))
                if bias.shape != (co,):
                    g.fail('%s: bias of shape %s' % (conv.name, bias.shape))
                hit = (r, w, bias)
                break
            if hit is None:
                g.fail('no conv%d in the %s branch' % (li + 1, ('pred', 'gt')[branch]))
            r, w, bias = hit
            _keep(out, g, 'w%d' % (li + 1), w)
            _keep(out, g, 'b%d' % (li + 1), bias)
            prev = r.name
            feats[branch].append(r.name)
    # distance head of layer l: Pow(Sub(f_pred / (norm + eps), f_gt / (norm + eps)), 2), then the 1x1 lin conv
    for li in range(5):
        head = None
        for n in g.nodes.values():
            if n.op != 'Pow' or g.inp(n, 0).op != 'Sub':
                continue
            a, b = g.inp(g.inp(n, 0), 0), g.inp(g.inp(n, 0), 1)
            if a.op == 'RealDiv' and b.op == 'RealDiv' and g.inp(a, 0).name == feats[0][li] and \
                    g.inp(b, 0).name == feats[1][li]:
                head = n
                break
        if head is None:
            g.fail('no distance head for layer %d' % (li + 1))
        if float(g.value(g.inp(head, 1), ())) != 2.0:
            g.fail('%s: exponent is not 2' % head.name)
        for dv in (a, b):
            eps = g.inp(dv, 1, 'Add')
            if float(g.value(g.inp(eps, 1), ())) != np.float32(1e-10):
                g.fail('%s: epsilon is not 1e-10' % eps.name)
        C = ALEX[li][0]
        lin = None
        for m in g.nodes.values():
            if m.op == 'Conv2D' and g.inp(m, 0).op == 'Split':
                pad = g.transpose(g.inp(g.inp(m, 0), 1), NCHW_TO_NHWC) if g.inp(g.inp(m, 0), 1).op == 'Transpose' \
                    else None
                if pad is not None and pad.op == 'Pad' and g.inp(pad, 0).name == head.name:
                    _, p, w = g.conv(m, 1, (1, C, 1, 1))
                    if p != 0:
                        g.fail('%s: padded lin conv' % m.name)
                    lin = w.reshape(C)
        if lin is None:
            g.fail('no lin conv for layer %d' % (li + 1))
        if (lin < 0).any():
            g.fail('lin%d has negative weights' % (li + 1))
        out['lin%d' % (li + 1)] = lin
    return {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in out.items()}
