"""Host-side execution engine for the NLT UV-space hot path.

A small explicit tape (no torch.autograd): every fused op records its own
backward closure; gradient buffers are accumulated in place by the dgrad
kernels (beta) and the activation-derivative mask is applied by the LAST
contributor, so no separate add / mask passes ever run.  All arithmetic is
done by the CUDA library behind include/nlt_b200.h; torch is used only for
device memory and streams.
"""
import ctypes as C
import math
import os

import torch

import nlt_native as nat


class Profiler:
    """Optional per-call device timing (bench.py's roofline leg): CUDA events
    on the launching stream around each C-ABI call, keyed by a label, with the
    call's algorithmic bytes.  Disabled (zero overhead) unless `enabled`."""

    def __init__(self):
        self.enabled = False
        self.records = []     # (label, bytes, start_event, end_event)

    def run(self, label, nbytes, fn):
        if not self.enabled:
            return fn()
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn()
        e1.record()
        self.records.append((label, nbytes, e0, e1))
        return r

    def summary(self):
        torch.cuda.synchronize()
        agg = {}
        for label, nbytes, e0, e1 in self.records:
            a = agg.setdefault(label, [0, 0.0, 0])
            a[0] += 1
            a[1] += e0.elapsed_time(e1)
            a[2] += nbytes
        self.records = []
        return {k: {'launches': v[0], 'ms': v[1], 'bytes': v[2]} for k, v in agg.items()}


PROF = Profiler()


def same_pad(n, k, s):
    """TF 'SAME' (pad_before, pad_after) -- see SURVEY.md section 8c."""
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


class Act:
    """An activation tensor [N,H,W,C] plus the bookkeeping of its gradient."""
    __slots__ = ('t', 'act', 'grad', 'n_cons', 'n_contrib', 'needs_grad', 'pending')

    def __init__(self, t, act=None, needs_grad=False):
        self.t = t
        self.act = act            # activation that produced t (mask source)
        self.grad = None
        self.n_cons = 0           # consumers that will contribute a gradient
        self.n_contrib = 0
        self.needs_grad = needs_grad
        self.pending = None       # deferred pointwise contribution: (PwTerm, keep-alive tensors, write_fn)


class Seg:
    """One source of a virtual channel concat."""
    __slots__ = ('a', 'sub', 'bcast')

    def __init__(self, a, sub=None, bcast=False):
        self.a = a if isinstance(a, Act) else Act(a)
        self.sub = sub
        self.bcast = bcast

    @property
    def C(self):
        return self.a.t.shape[3]


class Tape:
    def __init__(self):
        self.ops = []

    def record(self, fn):
        self.ops.append(fn)

    def backward(self):
        for fn in reversed(self.ops):
            fn()
        if USE_SIDE_STREAM and torch.cuda.is_available():
            # join the weight-gradient branches BEFORE the closures (and with them the activations the side streams
            # may still be reading) are released
            for i in range(N_SIDE_STREAMS):
                torch.cuda.current_stream().wait_stream(side_stream(i))
        self.ops = []
        while _PARKED:                      # leaves whose parked contribution nobody took along
            settle(_PARKED.pop())


class PackArena:
    """Bump allocator for the packed weight planes of ONE step (hi / lo TF32 planes of every tensor-core layer call):
    with PACK_AHEAD the planes are produced on the pack stream ahead of the layers that read them, so every call needs
    its own buffer.  Chunks are kept (addresses stay valid for a captured graph); `reset()` rewinds at step begin."""
    CHUNK = 256 << 20

    def __init__(self):
        self.chunks = []
        self.ci = 0
        self.off = 0

    def reset(self):
        self.ci = 0
        self.off = 0

    def alloc(self, nbytes, device):
        """A float32 view of at least `nbytes` bytes, 256-byte aligned inside its chunk."""
        n = (nbytes + 255) // 256 * 64                      # floats
        while True:
            if self.ci < len(self.chunks):
                buf = self.chunks[self.ci]
                if buf.device == device and self.off + n <= buf.numel():
                    out = buf[self.off:self.off + n]
                    self.off += n
                    return out
                self.ci += 1
                self.off = 0
                continue
            self.chunks.append(torch.empty(max(self.CHUNK // 4, n), dtype=torch.float32, device=device))


class Workspace:
    """Grow-only device scratch shared by all wgrad calls on one stream."""

    def __init__(self):
        self.buf = None
        self.subs = {}
        self.arena = PackArena()

    def sub(self, i):
        """Scratch of the i-th weight-gradient stream (0: this object)."""
        if i == 0:
            return self
        if i not in self.subs:
            self.subs[i] = Workspace()
        return self.subs[i]

    def get(self, nbytes, device):
        if self.buf is None or self.buf.numel() * 4 < nbytes or self.buf.device != device:
            self.buf = torch.empty((max(nbytes, 1 << 20) + 3) // 4, dtype=torch.float32, device=device)
        return self.buf


_WS = Workspace()
_WS_SIDE = Workspace()       # scratch of the weight-gradient stream


class use_workspaces:
    """Context manager: route the scratch requests of every op issued inside it to the given Workspace pair.
    A captured CUDA graph bakes the raw scratch addresses into its kernel arguments (packed hi/lo weight planes,
    TMA maps, wgrad partials), so a graph must own its scratch: trainvali.GraphedTrainStep warms up and captures
    inside `use_workspaces(own_main, own_side)` and keeps both objects alive as long as the graph.  A later eager
    call that needs a larger scratch grows the module-level pair only, never the graph's."""

    def __init__(self, main, side):
        self.pair = (main, side)

    def __enter__(self):
        global _WS, _WS_SIDE
        self.saved = (_WS, _WS_SIDE)
        _WS, _WS_SIDE = self.pair
        return self

    def __exit__(self, *exc):
        global _WS, _WS_SIDE
        _WS, _WS_SIDE = self.saved
        return False
_SIDE = {}                   # (device index, i) -> side stream
# weight-gradient streams (NLT_SIDE_STREAMS, default 2): consecutive layers' weight gradients go round-robin to
# different streams, so that the latency-bound launches of the deep levels overlap each other too
N_SIDE_STREAMS = max(1, int(os.environ.get('NLT_SIDE_STREAMS', '2')))
_side_rr = [0]


def side_stream(i=0):
    """Weight gradients do not feed the input-gradient chain: they run on a second stream (a parallel
    branch of the captured CUDA graph), which hides the launch/latency-bound deep-level launches behind
    the main chain.  Joined back in Tape.backward()."""
    dev = torch.cuda.current_device()
    if (dev, i) not in _SIDE:
        _SIDE[(dev, i)] = torch.cuda.Stream(device=dev)
    return _SIDE[(dev, i)]


def join_side_streams():
    """Orders side stream 0 after everything issued so far on the other weight-gradient streams."""
    for i in range(1, N_SIDE_STREAMS):
        side_stream(0).wait_stream(side_stream(i))


USE_SIDE_STREAM = os.environ.get('NLT_NO_SIDE_STREAM', '0') != '1'
_SKIP_WGRAD = os.environ.get('NLT_SKIP_WGRAD', '0') == '1'
# called as WGRAD_HOOK(layer) right after a layer's weight-gradient launch has been issued (on the side stream when
# USE_SIDE_STREAM): trainvali.GradReducer starts the early part of the gradient all-reduce from it
WGRAD_HOOK = None
# debugging / parity tap: FWD_TAP(layer, output tensor) after every conv launch (tests/test_gpu_parity.py collects the
# activation-derivative masks of the product with it)
FWD_TAP = None


# NLT_PACK_AHEAD (default 0): weight planes of the tensor-core layers are packed on a stream that hangs off the START
# of the step (weights are final there) instead of in front of each layer's kernel on the main stream.  Inside the
# captured CUDA graph the pack nodes do not start earlier than before, and eager launches pay the extra stream switches
# on the host -- so the switch stays off; the C-ABI entry points and the scheduling-invariance test remain.
PACK_AHEAD = os.environ.get('NLT_PACK_AHEAD', '0') == '1'
_PACK = {}                   # device index -> pack stream
_STEP_ROOT = {}              # device index -> [event recorded on the main stream at step begin, forked?]


def pack_stream():
    dev = torch.cuda.current_device()
    if dev not in _PACK:
        _PACK[dev] = torch.cuda.Stream(device=dev)
    return _PACK[dev]


def begin_step():
    """Marks the start of a forward (+ backward) pass: everything the pack stream does in this step depends on this
    point only.  Called by the model before its first layer."""
    if not (PACK_AHEAD and torch.cuda.is_available()):
        return
    _WS.arena.reset()
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream())
    _STEP_ROOT[torch.cuda.current_device()] = [ev, False]


def gconv_fwd(d, bias, act, beta, mask, mask_act, out):
    """nlt_gconv_fwd_ws with the shared scratch (tensor-core path where the
    shape allows it, fp32 kernels otherwise)."""
    lib = nat.lib()
    root = _STEP_ROOT.get(out.device.index) if PACK_AHEAD else None
    if root is not None:
        pb = lib.nlt_gconv_fwd_pack_bytes(C.byref(d), beta, 1 if mask is not None else 0)
        if pb < 0:
            nat.check(-1)
        if pb > 0:
            main, ps = torch.cuda.current_stream(), pack_stream()
            if not root[1]:
                ps.wait_event(root[0])                   # fork off the start of the step
                root[1] = True
            buf = _WS.arena.alloc(pb, out.device)
            with torch.cuda.stream(ps):
                nat.check(lib.nlt_gconv_pack_weights(C.byref(d), nat.ptr(buf), buf.numel() * 4, nat.stream()))
            main.wait_stream(ps)
            nat.check(lib.nlt_gconv_fwd_packed(C.byref(d), nat.ptr(bias), act, beta, nat.ptr(mask), mask_act,
                                               nat.ptr(out), nat.ptr(buf), buf.numel() * 4, nat.stream()))
            return
    need = lib.nlt_gconv_fwd_workspace_bytes(C.byref(d))
    if need < 0:
        nat.check(-1)
    if need > 0:
        ws = _WS.get(need, out.device)
        nat.check(lib.nlt_gconv_fwd_ws(C.byref(d), nat.ptr(bias), act, beta, nat.ptr(mask), mask_act, nat.ptr(out),
                                       nat.ptr(ws), ws.numel() * 4, nat.stream()))
    else:
        nat.check(lib.nlt_gconv_fwd_ws(C.byref(d), nat.ptr(bias), act, beta, nat.ptr(mask), mask_act, nat.ptr(out),
                                       None, 0, nat.stream()))


FUSE_POINTWISE_DGRAD = os.environ.get('NLT_FUSE_DGRAD', '1') != '0'
_PARKED = []     # Acts holding a parked contribution (settled at the latest when the tape finishes)


def contribute(target, write_fn, offer=None, can_fuse=None):
    """Adds one gradient contribution into target.grad.
    write_fn(out, beta, mask_y, mask_act, term) launches the producing kernel (term: a PwTerm to add in the
    kernel's epilogue, or None).

    offer = (PwTerm, keep-alive tensors): this contribution IS a small pointwise product (the input gradient
    of the final 1x1 conv).  When it would be the first of several it is not launched but parked on the
    target; the next contributor adds it in its own epilogue if its kernel can (can_fuse(term, out, mask) ->
    bool, backed by nlt_gconv_fwd_fused_supported) -- the full-resolution gradient tensor is then written
    once instead of written, re-read and re-written.  Otherwise the parked one is issued first, as usual."""
    if target.pending is not None:
        pterm, _keep, pwrite = target.pending
        target.pending = None
        target.grad = torch.empty_like(target.t)        # parked => nothing has been written yet
        target.n_contrib += 1
        last = target.n_contrib == target.n_cons
        mask = target.t if (last and target.act is not None) else None
        mask_act = nat.ACT_CODES[target.act] if mask is not None else 0
        if can_fuse is not None and can_fuse(pterm, target.grad, mask):
            write_fn(target.grad, 0.0, mask, mask_act, pterm)
        else:
            pwrite(target.grad, 0.0, None, 0, None)
            write_fn(target.grad, 1.0, mask, mask_act, None)
        return
    if (FUSE_POINTWISE_DGRAD and offer is not None and target.grad is None
            and target.n_cons - target.n_contrib >= 2):
        target.pending = (offer[0], offer[1], write_fn)
        target.n_contrib += 1
        _PARKED.append(target)
        return
    if target.grad is None:
        target.grad = torch.empty_like(target.t)
        beta = 0.0
    else:
        beta = 1.0
    target.n_contrib += 1
    last = target.n_contrib == target.n_cons
    mask = target.t if (last and target.act is not None) else None
    write_fn(target.grad, beta, mask, nat.ACT_CODES[target.act] if mask is not None else 0, None)


def settle(a):
    """Issues a parked contribution of `a` on its own (no later contributor took it along)."""
    if a.pending is not None:
        _pterm, _keep, pwrite = a.pending
        a.pending = None
        a.grad = torch.empty_like(a.t)
        last = a.n_contrib == a.n_cons
        mask = a.t if (last and a.act is not None) else None
        pwrite(a.grad, 0.0, mask, nat.ACT_CODES[a.act] if mask is not None else 0, None)


class ConvLayer:
    """One Conv2D / Conv2DTranspose ('same', bias) with a fused activation.
    Reference: nlt/networks/elements.py:26-39 (+ :69-78 for the activation).
    Kernel layouts are Keras': conv (kh,kw,Ci,Co), deconv (kh,kw,Co,Ci)."""

    def __init__(self, kind, k, s, cout, act=None):
        assert kind in ('conv', 'deconv')
        self.kind, self.k, self.s, self.cout, self.act = kind, k, s, cout, act
        self.cin = None
        self.name = '%s%dx%d/s%d->%d' % (kind, k, k, s, cout)
        self.kernel = self.bias = self.gkernel = self.gbias = None
        self.grad_written = False

    # ---- parameters -------------------------------------------------------
    def kernel_shape(self, cin):
        k = self.k
        return (k, k, cin, self.cout) if self.kind == 'conv' else (k, k, self.cout, cin)

    @property
    def built(self):
        return self.kernel is not None

    def build(self, cin, device, generator=None):
        """Keras defaults: Glorot-uniform kernel, zero bias."""
        self.cin = cin
        shape = self.kernel_shape(cin)
        limit = math.sqrt(6.0 / (self.k * self.k * (cin + self.cout)))
        w = (torch.rand(shape, generator=generator, dtype=torch.float32) * 2 - 1) * limit
        self.kernel = w.to(device)
        self.bias = torch.zeros(self.cout, dtype=torch.float32, device=device)
        self.gkernel = torch.zeros_like(self.kernel)
        self.gbias = torch.zeros_like(self.bias)

    # ---- descriptors ------------------------------------------------------
    def _geometry(self, Hin, Win):
        k, s = self.k, self.s
        if self.kind == 'conv':
            Hout, Wout = -(-Hin // s), -(-Win // s)
            pt, pl = same_pad(Hin, k, s)[0], same_pad(Win, k, s)[0]
        else:
            Hout, Wout = Hin * s, Win * s
            pt, pl = same_pad(Hout, k, s)[0], same_pad(Wout, k, s)[0]
        return Hout, Wout, pt, pl

    def _fwd_desc(self, segs, N, Hin, Win):
        Hout, Wout, pt, pl = self._geometry(Hin, Win)
        d = nat.GConvDesc()
        d.N, d.Hin, d.Win, d.Hout, d.Wout = N, Hin, Win, Hout, Wout
        d.kh = d.kw = self.k
        d.stride, d.pad_t, d.pad_l = self.s, pt, pl
        d.transposed = 0 if self.kind == 'conv' else 1
        d.nseg = len(segs)
        for i, sg in enumerate(segs):
            d.seg_ptr[i] = nat.ptr(sg.a.t)
            d.seg_sub[i] = nat.ptr(sg.sub)
            d.seg_C[i] = sg.C
            d.seg_bcast[i] = 1 if sg.bcast else 0
        d.Cout = self.cout
        d.w = nat.ptr(self.kernel)
        ci, co = self.cin, self.cout
        if self.kind == 'conv':
            d.w_tap_stride, d.w_c_stride, d.w_n_stride = ci * co, co, 1
        else:
            d.w_tap_stride, d.w_c_stride, d.w_n_stride = ci * co, 1, ci
        return d

    def _dgrad_desc(self, dz, N, Hin, Win, coff, cseg):
        """Adjoint op producing d(input segment) from dz = d(pre-activation out)."""
        Hout, Wout, pt, pl = self._geometry(Hin, Win)
        d = nat.GConvDesc()
        d.N, d.Hin, d.Win, d.Hout, d.Wout = N, Hout, Wout, Hin, Win
        d.kh = d.kw = self.k
        d.stride, d.pad_t, d.pad_l = self.s, pt, pl
        d.transposed = 1 if self.kind == 'conv' else 0
        d.nseg = 1
        d.seg_ptr[0] = nat.ptr(dz)
        d.seg_sub[0] = None
        d.seg_C[0] = self.cout
        d.seg_bcast[0] = 0
        d.Cout = cseg
        ci, co = self.cin, self.cout
        base = self.kernel.data_ptr()
        if self.kind == 'conv':      # (kh,kw,Ci,Co): contraction over Co, output over Ci
            d.w = base + 4 * coff * co
            d.w_tap_stride, d.w_c_stride, d.w_n_stride = ci * co, 1, co
        else:                        # (kh,kw,Co,Ci)
            d.w = base + 4 * coff
            d.w_tap_stride, d.w_c_stride, d.w_n_stride = ci * co, ci, 1
        return d

    # ---- execution --------------------------------------------------------
    def forward(self, segs, tape=None):
        lib = nat.lib()
        ref = next(sg for sg in segs if not sg.bcast).a.t
        N, Hin, Win = ref.shape[0], ref.shape[1], ref.shape[2]
        cin = sum(sg.C for sg in segs)
        if not self.built:
            self.build(cin, ref.device)
        if cin != self.cin:
            raise ValueError('layer built for %d input channels, got %d' % (self.cin, cin))
        for sg in segs:
            t = sg.a.t
            if t.shape[1] != Hin or t.shape[2] != Win or (not sg.bcast and t.shape[0] != N) \
                    or (sg.bcast and t.shape[0] != 1):
                raise ValueError('segment shape %s incompatible with %s' % (tuple(t.shape), tuple(ref.shape)))
        d = self._fwd_desc(segs, N, Hin, Win)
        out = torch.empty((N, d.Hout, d.Wout, self.cout), dtype=torch.float32, device=ref.device)
        nb = 4 * (sum(sg.a.t.numel() * (2 if sg.sub is not None else 1) for sg in segs) + out.numel())
        PROF.run('fwd ' + self.name, nb, lambda: gconv_fwd(d, self.bias, nat.ACT_CODES[self.act], 0.0, None, 0, out))
        if FWD_TAP is not None:
            FWD_TAP(self, out)
        y = Act(out, act=self.act, needs_grad=tape is not None)
        if tape is not None:
            for sg in segs:
                if sg.a.needs_grad:
                    sg.a.n_cons += 1
            tape.record(lambda: self._backward(segs, y, N, Hin, Win))
        return y

    def _backward(self, segs, y, N, Hin, Win):
        lib = nat.lib()
        settle(y)
        dz = y.grad
        if dz is None:
            return
        # weight / bias gradient (same descriptor as forward, G = dz)
        d = self._fwd_desc(segs, N, Hin, Win)
        need = lib.nlt_gconv_wgrad_workspace_bytes(C.byref(d))
        if need < 0:
            nat.check(-1)
        nb = 4 * (sum(sg.a.t.numel() * (2 if sg.sub is not None else 1) for sg in segs) + dz.numel())
        acc = 1 if self.grad_written else 0
        if _SKIP_WGRAD:          # DIAGNOSTIC (NLT_SKIP_WGRAD=1, wrong results): time the forward + input-gradient chain alone
            pass
        elif USE_SIDE_STREAM:
            if getattr(self, '_side_idx', None) is None or self._side_idx >= N_SIDE_STREAMS:
                self._side_idx = _side_rr[0] % N_SIDE_STREAMS      # one stream per layer: repeated (accumulating)
                _side_rr[0] += 1                                   # launches of a layer stay ordered
            si = self._side_idx
            main, side = torch.cuda.current_stream(), side_stream(si)
            side.wait_stream(main)                      # dz (and the inputs) are complete on the main stream
            with torch.cuda.stream(side):
                ws = _WS_SIDE.sub(si).get(need, dz.device)
                PROF.run('wgrad ' + self.name, nb, lambda: nat.check(lib.nlt_gconv_wgrad(
                    C.byref(d), nat.ptr(dz), nat.ptr(self.gkernel), nat.ptr(self.gbias), acc, nat.ptr(ws),
                    ws.numel() * 4, nat.stream())))
            dz.record_stream(side)                      # dz is released below while the side stream may still read it
        else:
            ws = _WS.get(need, dz.device)
            PROF.run('wgrad ' + self.name, nb, lambda: nat.check(lib.nlt_gconv_wgrad(
                C.byref(d), nat.ptr(dz), nat.ptr(self.gkernel), nat.ptr(self.gbias), acc, nat.ptr(ws),
                ws.numel() * 4, nat.stream())))
        self.grad_written = True
        if WGRAD_HOOK is not None:
            WGRAD_HOOK(self)
        # input gradients, one adjoint launch per differentiable segment
        pointwise = self.kind == 'conv' and self.k == 1 and self.s == 1 and self.cout <= 4
        coff = 0
        for sg in segs:
            if sg.a.needs_grad:
                dd = self._dgrad_desc(dz, N, Hin, Win, coff, sg.C)

                def write(out, beta, mask, mask_act, term, dd=dd):
                    nb = 4 * (dz.numel() + out.numel() * (1 + (beta != 0) + (mask is not None)))
                    if term is None:
                        PROF.run('dgrad ' + self.name, nb, lambda: gconv_fwd(dd, None, 0, beta, mask, mask_act, out))
                    else:
                        PROF.run('dgrad ' + self.name, nb, lambda: nat.check(lib.nlt_gconv_fwd_fused(
                            C.byref(dd), C.byref(term), None, 0, beta, nat.ptr(mask), mask_act, nat.ptr(out),
                            nat.stream())))

                def can_fuse(term, out, mask, dd=dd):
                    return bool(lib.nlt_gconv_fwd_fused_supported(C.byref(dd), C.byref(term), nat.ptr(mask),
                                                                  nat.ptr(out)))
                offer = None
                if pointwise:
                    # d(input)[p, c] = sum_co dz[p, co] * W[coff + c, co]   (kernel layout (1,1,Ci,Co))
                    term = nat.PwTerm()
                    term.x, term.K = nat.ptr(dz), self.cout
                    term.w = self.kernel.data_ptr() + 4 * coff * self.cout
                    term.w_k_stride, term.w_n_stride = 1, self.cout
                    offer = (term, (dz, self.kernel))
                contribute(sg.a, write, offer, can_fuse)
            coff += sg.C
        y.grad = None   # dz is dead: release it


class NormLayer:
    """`norm(type)` + the activation that follows it in a block (nlt/networks/convnet.py:50-59, 67-76):
    'pixel' (elements.py:103-121, no parameters) or 'instance' (elements.py:97-100: per-sample, per-channel
    statistics over H x W, eps 1e-6, learnable scale `kernel` (gamma, ones) and centre `bias` (beta, zeros)).
    The conv in front of it runs without activation; this op applies norm and activation in one pass and its
    backward turns d(norm output) into d(conv output)."""
    EPS_INSTANCE = 1.0e-6

    def __init__(self, kind, act=None):
        assert kind in ('pixel', 'instance')
        self.kind, self.act = kind, act
        self.has_params = kind == 'instance'
        self.cout = None
        self.name = kind + 'norm'
        self.kernel = self.bias = self.gkernel = self.gbias = None
        self.grad_written = False
        self._ws = None

    @property
    def built(self):
        return self.cout is not None

    def build(self, C, device, generator=None):
        self.cout = C
        if self.has_params:
            self.kernel = torch.ones(C, dtype=torch.float32, device=device)
            self.bias = torch.zeros(C, dtype=torch.float32, device=device)
            self.gkernel, self.gbias = torch.zeros_like(self.kernel), torch.zeros_like(self.bias)
        return C

    def _workspace(self, N, HW, C, device):
        need = nat.lib().nlt_instnorm_workspace_bytes(N, HW, C)
        if need < 0:
            nat.check(-1)
        if self._ws is None or self._ws.numel() * 4 < need or self._ws.device != device:
            self._ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=device)
        return self._ws

    def forward(self, x, tape=None):
        lib = nat.lib()
        t = x.t
        N, H, W, C = t.shape
        if not self.built:
            self.build(C, t.device)
        if C != self.cout:
            raise ValueError('norm built for %d channels, got %d' % (self.cout, C))
        y = torch.empty_like(t)
        act = nat.ACT_CODES[self.act]
        saved = None
        if self.kind == 'pixel':
            PROF.run('fwd ' + self.name, 8 * t.numel(), lambda: nat.check(
                lib.nlt_pixelnorm_fwd(nat.ptr(t), N * H * W, C, act, nat.ptr(y), nat.stream())))
        else:
            mean = torch.empty(N * C, dtype=torch.float32, device=t.device)
            rstd = torch.empty_like(mean)
            ws = self._workspace(N, H * W, C, t.device)
            PROF.run('fwd ' + self.name, 12 * t.numel(), lambda: nat.check(lib.nlt_instnorm_fwd(
                nat.ptr(t), nat.ptr(self.kernel), nat.ptr(self.bias), N, H * W, C, act, self.EPS_INSTANCE, nat.ptr(y),
                nat.ptr(mean), nat.ptr(rstd), nat.ptr(ws), nat.stream())))
            saved = (mean, rstd)
        out = Act(y, act=self.act, needs_grad=tape is not None)
        if tape is not None:
            if x.needs_grad:
                x.n_cons += 1
            tape.record(lambda: self._backward(x, out, saved))
        return out

    def _backward(self, x, out, saved):
        lib = nat.lib()
        settle(out)
        dz = out.grad
        if dz is None or not x.needs_grad:
            return
        t = x.t
        N, H, W, C = t.shape

        def write(o, beta, mask, mask_act, term):
            # the conv in front has no activation of its own and this op is its only consumer
            assert beta == 0.0 and mask is None and term is None
            if self.kind == 'pixel':
                PROF.run('dgrad ' + self.name, 12 * t.numel(), lambda: nat.check(
                    lib.nlt_pixelnorm_bwd(nat.ptr(t), nat.ptr(dz), N * H * W, C, nat.ptr(o), nat.stream())))
            else:
                mean, rstd = saved
                ws = self._workspace(N, H * W, C, t.device)
                acc = 1 if self.grad_written else 0
                PROF.run('dgrad ' + self.name, 20 * t.numel(), lambda: nat.check(lib.nlt_instnorm_bwd(
                    nat.ptr(t), nat.ptr(dz), nat.ptr(self.kernel), nat.ptr(mean), nat.ptr(rstd), N, H * W, C, nat.ptr(o),
                    nat.ptr(self.gkernel), nat.ptr(self.gbias), acc, nat.ptr(ws), nat.stream())))
                self.grad_written = True
        contribute(x, write)
        out.grad = None


class PoolLayer:
    """`pool(type)` at the end of a down block (nlt/networks/elements.py:81-94, convnet.py:58): 2x2 / stride-2 'same'
    max or average pooling.  The output carries no activation; the backward pass makes one contribution into its
    input, which applies that input's activation mask.  The max argmax is recomputed from the input, which is kept
    anyway as the mask source, so nothing new is stored."""
    KINDS = {'max': 0, 'avg': 1}          # NLT_POOL_MAX / NLT_POOL_AVG

    def __init__(self, kind):
        assert kind in self.KINDS
        self.kind = kind
        self.name = kind + 'pool'

    def forward(self, x, tape=None):
        lib = nat.lib()
        t = x.t
        N, H, W, C = t.shape
        y = torch.empty((N, (H + 1) // 2, (W + 1) // 2, C), dtype=torch.float32, device=t.device)
        code = self.KINDS[self.kind]
        PROF.run('fwd ' + self.name, 4 * (t.numel() + y.numel()), lambda: nat.check(
            lib.nlt_pool2x2_fwd(nat.ptr(t), N, H, W, C, code, nat.ptr(y), nat.stream())))
        out = Act(y, act=None, needs_grad=tape is not None and x.needs_grad)
        if tape is not None and x.needs_grad:
            x.n_cons += 1

            def bwd():
                settle(out)
                dy = out.grad
                if dy is None:
                    return

                def write(o, beta, mask, mask_act, term=None):
                    nb = 4 * (dy.numel() + o.numel() * (2 + (beta != 0) + (mask is not None)))
                    PROF.run('dgrad ' + self.name, nb, lambda: nat.check(lib.nlt_pool2x2_bwd(
                        nat.ptr(t), nat.ptr(dy), N, H, W, C, code, beta, nat.ptr(mask), mask_act, nat.ptr(o),
                        nat.stream())))
                contribute(x, write)
                out.grad = None
            tape.record(bwd)
        return out


def upsample2x(a, tape=None):
    """UpSampling2D(2, 'bilinear') of one Act (the first half of `upconv`, nlt/networks/elements.py:42-48).  A batch-1
    broadcast source stays batch 1.  The result's gradient accumulates from every segment that reads it; its backward
    pass then makes one contribution into the source."""
    lib = nat.lib()
    t = a.t
    N, H, W, C = t.shape
    y = torch.empty((N, 2 * H, 2 * W, C), dtype=torch.float32, device=t.device)
    PROF.run('fwd upsample2x', 4 * (t.numel() + y.numel()), lambda: nat.check(
        lib.nlt_upsample2x_bilinear_fwd(nat.ptr(t), N, H, W, C, nat.ptr(y), nat.stream())))
    out = Act(y, act=None, needs_grad=tape is not None and a.needs_grad)
    if tape is not None and a.needs_grad:
        a.n_cons += 1

        def bwd():
            settle(out)
            dy = out.grad
            if dy is None:
                return

            def write(o, beta, mask, mask_act, term=None):
                nb = 4 * (dy.numel() + o.numel() * (1 + (beta != 0) + (mask is not None)))
                PROF.run('dgrad upsample2x', nb, lambda: nat.check(lib.nlt_upsample2x_bilinear_bwd(
                    nat.ptr(dy), N, H, W, C, beta, nat.ptr(mask), mask_act, nat.ptr(o), nat.stream())))
            contribute(a, write)
            out.grad = None
        tape.record(bwd)
    return out


def kmean(obs_y, K, tape=None, weights=None):
    """mean over the K stacked observations (nlt/models/nlt.py:161-164).
    obs_y: Act [K*B,H,W,C] (k-major).  K == 1 aliases (no kernel, no copy)."""
    if K == 1 and weights is None:
        return obs_y
    lib = nat.lib()
    t = obs_y.t
    B = t.shape[0] // K
    per = t.shape[1] * t.shape[2] * t.shape[3]
    out = torch.empty((B,) + tuple(t.shape[1:]), dtype=torch.float32, device=t.device)
    PROF.run('fwd kmean', 4 * (t.numel() + out.numel()), lambda: nat.check(
        lib.nlt_kmean_fwd(nat.ptr(t), nat.ptr(weights), K, B, per, nat.ptr(out), nat.stream())))
    agg = Act(out, act=None, needs_grad=tape is not None and obs_y.needs_grad)
    if tape is not None and obs_y.needs_grad:
        obs_y.n_cons += 1

        def bwd():
            settle(agg)
            if agg.grad is None:
                return

            def write(o, beta, mask, mask_act, term=None):
                nb = 4 * (agg.grad.numel() + o.numel() * (1 + (beta != 0) + (mask is not None)))
                PROF.run('dgrad kmean', nb, lambda: nat.check(lib.nlt_kmean_bwd(
                    nat.ptr(agg.grad), nat.ptr(weights), K, B, per, beta, nat.ptr(mask), mask_act, nat.ptr(o),
                    nat.stream())))
            contribute(obs_y, write)
            agg.grad = None
        tape.record(bwd)
    return agg


class ParamBucket:
    """All trainable parameters of a model in ONE contiguous fp32 buffer (and
    one gradient buffer), so that the data-parallel step is a single fused
    AMSGrad launch and at most two all-reduce calls (nlt/trainvali.py:279-280).

    `layout`: order of the layers inside the flat buffers (default: as given).  models/nlt.py passes the order in
    which the backward pass PRODUCES the weight gradients (decoder top-down, then encoder levels bottom-up), so the
    gradient buffer fills front to back and its parameter-heavy head (the deep levels) can be all-reduced while the
    full-resolution levels are still running.  `grad` carries LOSS_SLOTS extra floats behind the parameters: the
    per-replica loss rides on the same collective (trainvali.py:317 is a second reduce in the reference)."""
    LOSS_SLOTS = 4

    def __init__(self, layers, device, layout=None):
        self.layers = list(layers)
        order = list(range(len(self.layers))) if layout is None else list(layout)
        assert sorted(order) == list(range(len(self.layers)))
        n = 0
        slices = [None] * len(self.layers)
        self.layout_ends = []                # (layer, end offset) in layout order
        for li in order:
            L = self.layers[li]
            assert L.built
            ks, bs = L.kernel.numel(), L.bias.numel()
            n_al = (n + 3) // 4 * 4          # keep every kernel 16B aligned
            slices[li] = (n_al, ks, n_al + ks, bs)
            n = n_al + ks + bs
            self.layout_ends.append((L, (n + 3) // 4 * 4))
        self.slices = slices
        self.n = (n + 3) // 4 * 4
        self.flat = torch.zeros(self.n, dtype=torch.float32, device=device)
        self._grad_all = torch.zeros(self.n + self.LOSS_SLOTS, dtype=torch.float32, device=device)
        self.grad = self._grad_all[:self.n]
        self.loss_slot = self._grad_all[self.n:self.n + 1]
        for L, (ko, ks, bo, bs) in zip(self.layers, self.slices):
            kshape, bshape = L.kernel.shape, L.bias.shape
            self.flat[ko:ko + ks].copy_(L.kernel.reshape(-1))
            self.flat[bo:bo + bs].copy_(L.bias.reshape(-1))
            L.kernel = self.flat[ko:ko + ks].view(kshape)
            L.bias = self.flat[bo:bo + bs].view(bshape)
            L.gkernel = self._grad_all[ko:ko + ks].view(kshape)
            L.gbias = self._grad_all[bo:bo + bs].view(bshape)

    def split_point(self, frac=0.9):
        """(layer, offset): the first layer boundary of the layout at which `frac` of the parameters lie in front;
        the collective of grad[:offset] may start as soon as that layer's weight gradient has been issued."""
        for L, end in self.layout_ends[:-1]:
            if end >= frac * self.n:
                return L, end
        return None, 0

    def grad_with_loss(self):
        """grad ++ loss slot: the buffer of the final collective."""
        return self._grad_all[:self.n + 1]

    def variables(self):
        out = []
        for L in self.layers:
            out += [L.kernel, L.bias]
        return out

    def gradients(self):
        out = []
        for L in self.layers:
            out += [L.gkernel, L.gbias]
        return out

    def begin_step(self):
        for L in self.layers:
            L.grad_written = False
