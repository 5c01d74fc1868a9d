"""NLT model on the CUDA hot path -- mirror of nlt/models/nlt.py:38-205.

Same surface as the reference: `Model(config)`, `register_trainable()`,
`model(batch, mode=)` == `model.call(batch, mode, obs_override=None)` ->
`(pred_camspc, gt_camspc, loss_kwargs, to_vis)`, `_call(query_x, obs_xs,
obs_weights, obs_override)`, `compute_loss(pred, gt, **kw)`, `.net` dict,
`.trainable_variables`.  The arithmetic is executed by hand-written sm_90a
kernels (include/nlt_b200.h) over a virtual channel concat: no tf.concat,
no `nn_rgb - nn_base`, no K-stack and no standalone bias/activation pass is
ever materialised.  Gradients are produced by `model.backward()` (the
reference uses tf.GradientTape in trainvali.py:272-281).
"""
import json
import os

import numpy as np
import torch

import losses
import nlt_native as nat
from engine import Act, Seg, Tape, ParamBucket, kmean, PROF
from networks import convnet
from .base import Model as BaseModel


def _dev_tensor(x, device, out=None):
    """Moves a batch element to the device as contiguous fp32 (inputs may be
    pinned host tensors: the H2D copy is part of the end-to-end path).
    uint8 tensors are image samples still in PNG units: they cross PCIe as bytes and become v / 255 on the device
    (bit-identical to the host pipeline's float32(v / 255.0); datasets with `uint8_inputs = True` emit them).
    `out`: a contiguous fp32 device tensor of the same shape to write into (the static inputs of a CUDA graph)."""
    if not torch.is_tensor(x):
        x = torch.as_tensor(np.asarray(x))
    if out is not None and (tuple(out.shape) != tuple(x.shape) or out.dtype != torch.float32 or not out.is_contiguous()):
        raise ValueError('batch element of shape %s / %s does not fit the fp32 buffer %s' % (
            tuple(x.shape), x.dtype, tuple(out.shape)))
    if x.dtype == torch.uint8:
        xd = x.to(device=device, non_blocking=True).contiguous()
        if out is None:
            out = torch.empty(xd.shape, dtype=torch.float32, device=device)
        nat.check(nat.lib().nlt_u8_to_f32(xd.data_ptr(), xd.numel(), nat.ptr(out), nat.stream()))
        return out
    if out is not None:
        return out.copy_(x, non_blocking=True)
    if x.device != device or x.dtype != torch.float32:
        x = x.to(device=device, dtype=torch.float32, non_blocking=True)
    return x.contiguous()


class Model(BaseModel):
    def __init__(self, config):
        # Needed by Barron loss (kept for signature parity, nlt.py:41-42)
        self.imh = config.getint('DEFAULT', 'imh')
        self.imw = config.getint('DEFAULT', 'imw')
        super().__init__(config)
        depth0 = config.getint('DEFAULT', 'depth0')
        depth = config.getint('DEFAULT', 'depth')
        kernel = config.getint('DEFAULT', 'kernel')
        stride = config.getint('DEFAULT', 'stride')
        norm = config.get('DEFAULT', 'norm')
        act = config.get('DEFAULT', 'act')
        pool = config.get('DEFAULT', 'pool')
        net_args = (depth0, depth, kernel, stride)
        net_kwargs = {'norm_type': norm, 'act_type': act, 'pool_type': pool}
        self.net = {
            'query': convnet.Network(*net_args, **net_kwargs),
            'obs': convnet.Network(*net_args, **net_kwargs)}
        self.net['obs'].layers = [
            x for i, x in enumerate(self.net['obs'].layers)
            if self.net['obs'].is_contracting[i]]  # remove decoding layers
        self.uvh = self.config.getint('DEFAULT', 'uvh')
        self.uvw = self.config.getint('DEFAULT', 'uvw')
        self.device = torch.device('cuda', torch.cuda.current_device()) \
            if torch.cuda.is_available() else None
        self.seed = 0
        self._bucket = None
        self._tape = None
        self._d_pred = None
        self._loss_grad_scale = None
        self._scatter_ws = None

    # ------------------------------------------------------------------
    # parameters
    # ------------------------------------------------------------------
    def build(self, c_query=5, c_obs=3):
        """Creates every kernel/bias (Keras defaults: Glorot-uniform / zeros)
        inside ONE flat bucket.  The reference builds lazily on first call;
        so does this class (call() invokes build with the batch's channels)."""
        if self._bucket is not None:
            return
        if self.device is None:
            raise nat.NativeError('no CUDA device: the NLT hot path has no CPU fallback')
        nat.lib()   # fail loudly if the extension is missing
        use_obs = self.config.getboolean('DEFAULT', 'use_obs')
        gen = torch.Generator().manual_seed(self.seed)
        q_in, o_in, skips = c_query, c_obs, []
        q, o = self.net['query'], self.net['obs']
        for li, (blk, contr) in enumerate(zip(q.layers, q.is_contracting)):
            if contr:
                o_in = o.layers[li].build(o_in, self.device, gen)
                n = blk.build(q_in, self.device, gen)
                q_in = n + (o_in if use_obs else 0)
                skips.append(q_in)
            else:
                if skips:
                    q_in += skips.pop()
                q_in = blk.build(q_in, self.device, gen)
        # everything that owns parameters (convs, and the norm layers of `norm = instance`), in registration order
        layers = q.param_layers() + o.param_layers()
        # flat layout = the order in which backward() produces the weight gradients: decoder blocks top-down, then
        # per encoder level (bottom-up) the query block followed by the observation block, last layer first
        index = {id(c): i for i, c in enumerate(layers)}
        produced = []
        n_q = len(q.layers)
        for li in range(n_q - 1, -1, -1):
            produced += [index[id(c)] for _, c in reversed(q.layers[li].param_layers())]
            if q.is_contracting[li]:
                produced += [index[id(c)] for _, c in reversed(o.layers[li].param_layers())]
        self._bucket = ParamBucket(layers, self.device, layout=produced)
        for name, c in self.named_convs():   # profiler labels: 'query.1.0 conv2x2/s2 32->16'
            if hasattr(c, 'kind') and c.kind in ('conv', 'deconv'):
                c.name = '%s %s%dx%d/s%d %d->%d' % (name, c.kind, c.k, c.k, c.s, c.cin, c.cout)
            else:
                c.name = '%s %snorm %d' % (name, c.kind, c.cout)
        for net in ('query', 'obs'):         # parameter-free norm layers get labels too
            for li, blk in enumerate(self.net[net].layers):
                for ci, nm in enumerate(blk.norms):
                    if nm is not None and not nm.has_params:
                        nm.name = '%s.%d.%d.norm %snorm %d' % (net, li, ci, nm.kind, nm.cout)
                if getattr(blk, 'pool', None) is not None:
                    blk.pool.name = '%s.%d.pool %spool %d' % (net, li, blk.pool.kind, blk.convs[-1].cout)

    @property
    def trainable_variables(self):
        assert self.trainable_registered, \
            "Register the trainable layers before using `trainable_variables`"
        return [] if self._bucket is None else self._bucket.variables()

    @property
    def gradients(self):
        return [] if self._bucket is None else self._bucket.gradients()

    @property
    def flat_params(self):
        return self._bucket.flat

    @property
    def flat_grads(self):
        return self._bucket.grad

    @property
    def bucket(self):
        return self._bucket

    def named_convs(self):
        """('query.3.0', ConvLayer) -- and ('query.3.0.norm', NormLayer) for `norm = instance`, whose scale / centre
        vectors ride in the `kernel` / `bias` slots -- in registration order."""
        out = []
        for net in ('query', 'obs'):
            for li, blk in enumerate(self.net[net].layers):
                for suffix, c in blk.param_layers():
                    out.append(('%s.%d.%s' % (net, li, suffix), c))
        return out

    def load_params(self, params):
        """params: {'query.3.0.kernel': tensor (Keras layout), '...bias': ...}"""
        for name, c in self.named_convs():
            c.kernel.copy_(params[name + '.kernel'].to(c.kernel.device, torch.float32))
            c.bias.copy_(params[name + '.bias'].to(c.bias.device, torch.float32))

    def export_params(self):
        out = {}
        for name, c in self.named_convs():
            out[name + '.kernel'] = c.kernel.detach().clone()
            out[name + '.bias'] = c.bias.detach().clone()
        return out

    def export_grads(self):
        out = {}
        for name, c in self.named_convs():
            out[name + '.kernel'] = c.gkernel.detach().clone()
            out[name + '.bias'] = c.gbias.detach().clone()
        return out

    # ------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------
    def call(self, batch, mode, obs_override=None):
        self._validate_mode(mode)
        id_, base, cvis, lvis, warp, rgb, rgb_camspc, nn_id, nn_base, \
            nn_rgb, nn_rgb_camspc = batch  # *rgb* are placeholders for testing
        if self.device is None:
            raise nat.NativeError('no CUDA device: the NLT hot path has no CPU fallback')
        self._check_uv_size(base.shape[1], base.shape[2])
        dev = self.device
        base, cvis, lvis, warp = (_dev_tensor(t, dev) for t in (base, cvis, lvis, warp))
        # The reference passes exactly one neighbour (nlt.py:96, "only one neighbor") while `_call` takes a list of
        # K; here K observations may ride in the same two slots of the tuple, either as lists of K [B,H,W,3]
        # tensors or as one k-major [K,B,H,W,3] tensor each (SURVEY 8d cfg3: K = 6)
        if isinstance(nn_rgb, (list, tuple)):
            nn_rgb = torch.stack([_dev_tensor(t, dev) for t in nn_rgb], dim=0)
            nn_base = torch.stack([_dev_tensor(t, dev) for t in nn_base], dim=0)
        nn_base, nn_rgb = _dev_tensor(nn_base, dev), _dev_tensor(nn_rgb, dev)
        K = 1
        if nn_rgb.dim() == 5:
            K = nn_rgb.shape[0]
            if nn_base.shape != nn_rgb.shape or nn_rgb.shape[1] != base.shape[0]:
                raise ValueError('K-observation inputs must be [K,B,H,W,3], got %s / %s' % (
                    tuple(nn_rgb.shape), tuple(nn_base.shape)))
            nn_rgb = nn_rgb.reshape((-1,) + tuple(nn_rgb.shape[2:]))      # k-major stack: a view, no copy
            nn_base = nn_base.reshape((-1,) + tuple(nn_base.shape[2:]))
        train = mode == 'train'
        tape = Tape() if train else None
        import engine
        engine.begin_step()           # start of the step: what the weight-plane pack stream hangs off
        if train:
            self._bucket and self._bucket.begin_step()
        # x = concat(base, cvis, lvis); y_obs = [nn_rgb - nn_base]  (nlt.py:95-96)
        q_segs = [Seg(Act(base)), Seg(Act(cvis)), Seg(Act(lvis))]
        o_segs = [Seg(Act(nn_rgb), sub=nn_base)]
        net_out = self._call_segs(q_segs, o_segs, K, None, obs_override, tape)
        skip_connect_base = self.config.getboolean(
            'DEFAULT', 'skip_connect_base')
        # ---- UV -> camera tail (nlt.py:99-120) in one fused pass ----
        lib = nat.lib()
        B, H, W = base.shape[0], base.shape[1], base.shape[2]
        ih, iw = warp.shape[1], warp.shape[2]
        resize = (ih, iw) != (self.imh, self.imw)
        want_gt = mode in ('train', 'vali')
        if want_gt:
            rgb_camspc = _dev_tensor(rgb_camspc, dev)
        new = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        pred = new(B, H, W, 3)
        pred_c, base_c = new(B, ih, iw, 3), new(B, ih, iw, 3)
        fg_c = new(B, ih, iw, 3) if (resize and want_gt) else None
        gt_c = new(B, ih, iw, 3) if (want_gt and not resize) else None
        # algorithmic bytes of the tail: net_out + base in, pred out (UV); warp + rgb in, 4 gathers of 3 channels from
        # the two UV maps, pred/base/gt out (camera)
        tail_bytes = 4 * (9 * B * H * W + (2 + 6 + 3 * (1 if gt_c is not None else 0)
                                             + 3 * (2 + (gt_c is not None) + (fg_c is not None))) * B * ih * iw)
        PROF.run('fwd tail uv2cam', tail_bytes, lambda: nat.check(lib.nlt_uv2cam_fwd(
            nat.ptr(net_out.t), nat.ptr(base), nat.ptr(warp), nat.ptr(rgb_camspc) if gt_c is not None else None,
            B, H, W, ih, iw, 1 if skip_connect_base else 0, nat.ptr(pred), nat.ptr(pred_c), nat.ptr(base_c),
            nat.ptr(fg_c), nat.ptr(gt_c), nat.stream())))
        if resize:   # tf.image.resize to (imh, imw)  (nlt.py:116-120)
            def rs(x):
                y = new(B, self.imh, self.imw, 3)
                nat.check(lib.nlt_resize_bilinear_fwd(nat.ptr(x), B, ih, iw, 3, self.imh, self.imw, nat.ptr(y),
                                                      nat.stream()))
                return y
            pred_c, base_c = rs(pred_c), rs(base_c)
            if want_gt:
                fg_r = rs(fg_c)
                gt_c = new(B, self.imh, self.imw, 3)     # alpha_blend (nlt.py:132-133)
                nat.check(lib.nlt_mul(nat.ptr(rgb_camspc), nat.ptr(fg_r), gt_c.numel(), nat.ptr(gt_c), nat.stream()))
        if train:
            def tail_bwd():
                d = self._d_pred
                if d is None:
                    raise RuntimeError('backward() before compute_loss()')
                if resize:
                    d_full = new(B, ih, iw, 3)
                    nat.check(lib.nlt_resize_bilinear_bwd(nat.ptr(d), B, ih, iw, 3, self.imh, self.imw,
                                                          nat.ptr(d_full), nat.stream()))
                    d = d_full
                g = new(B, H, W, 3)
                # bit-reproducible scatter (64-bit fixed-point accumulation); its accumulator is zero-filled once
                # and handed back zero-filled by every call
                need = lib.nlt_uv2cam_bwd_workspace_bytes(B, H, W)
                if self._scatter_ws is None or self._scatter_ws.numel() * 8 < need or self._scatter_ws.device != dev:
                    self._scatter_ws = torch.zeros((need + 7) // 8, dtype=torch.int64, device=dev)
                ws = self._scatter_ws
                PROF.run('dgrad tail uv2cam', 4 * (5 * B * ih * iw + 3 * B * H * W), lambda: nat.check(
                    lib.nlt_uv2cam_bwd_det(nat.ptr(d), nat.ptr(warp), B, H, W, ih, iw, nat.ptr(g), ws.data_ptr(),
                                           nat.stream())))
                net_out.grad = g
            tape.record(tail_bwd)
        self._tape = tape
        self._d_pred = None
        to_vis = {
            'id': id_,
            'nn_id': nn_id,
            'base_camspc': base_c,
            'pred': pred,
            'pred_camspc': pred_c,
            'nn_camspc': nn_rgb_camspc}
        if want_gt:
            loss_kwargs = {}
            to_vis['gt'] = rgb
            to_vis['gt_camspc'] = gt_c
            return pred_c, gt_c, loss_kwargs, to_vis
        return pred_c, None, None, to_vis

    def _call(self, query_x, obs_xs, obs_weights=None, obs_override=None):
        """Reference signature (nlt.py:141): tensors in, tensor out."""
        self._check_uv_size(query_x.shape[1], query_x.shape[2])
        dev = self.device
        q = [Seg(Act(_dev_tensor(query_x, dev)))]
        K = len(obs_xs)
        obs = _dev_tensor(obs_xs[0], dev) if K == 1 else \
            torch.cat([_dev_tensor(x, dev) for x in obs_xs], dim=0)   # k-major stack
        if obs_weights is not None:
            obs_weights = _dev_tensor(obs_weights, dev).reshape(obs.shape[0] // K, K)
        return self._call_segs(q, [Seg(Act(obs))], K, obs_weights, obs_override, None).t

    def _check_uv_size(self, H, W):
        """With `pool` set every down block halves the UV map and the decoder concatenates each level's skip tensor at
        the same size, so H and W must be multiples of 2**(down blocks).  Raised before anything reaches the device."""
        n = sum(1 for blk in self.net['query'].layers if getattr(blk, 'pool', None) is not None)
        if n and (int(H) % (1 << n) or int(W) % (1 << n)):
            raise ValueError('pool=%s: the UV size %dx%d is not a multiple of 2**%d = %d (one halving per down block)'
                             % (self.net['query'].layers[1].pool.kind, int(H), int(W), n, 1 << n))

    def _call_segs(self, query_x, obs_x, K, obs_weights, obs_override, tape):
        """The two-stream U-Net walk of nlt.py:141-199 over virtual concats.
        query_x / obs_x: lists of engine.Seg; returns the last query_y (Act)."""
        use_obs = self.config.getboolean('DEFAULT', 'use_obs')
        self.build(sum(s.C for s in query_x), sum(s.C for s in obs_x))
        B = query_x[0].a.t.shape[0]
        # The reference runs the observation stream even when its result is
        # overridden / unused (nlt.py:151-164, 178-179); the outputs do not
        # depend on it, so it is skipped here in those cases.
        run_obs = use_obs and obs_override is None
        obs_tape = tape if run_obs else None
        query_featmaps = []
        query_y = None
        for layer_i, (layer_query, is_contracting) in enumerate(zip(
                self.net['query'].layers, self.net['query'].is_contracting)):
            if is_contracting:
                obs_agg = None
                if run_obs:
                    layer_obs = self.net['obs'].layers[layer_i]
                    obs_y = layer_obs.forward_segs(obs_x, obs_tape)   # all K observations, shared weights
                    obs_agg = Seg(kmean(obs_y, K, obs_tape, obs_weights))
                    obs_x = [Seg(obs_y)]      # don't concat the aggregate in the observation network
                query_y = layer_query.forward_segs(query_x, tape)
                if use_obs:
                    if obs_override is not None:
                        ov = _dev_tensor(obs_override[layer_i], self.device)
                        obs_agg = Seg(Act(ov), bcast=(ov.shape[0] == 1 and B > 1))
                    query_x = [Seg(query_y), obs_agg]
                else:
                    query_x = [Seg(query_y)]
                query_featmaps.append(query_x)
            else:
                # skip connections between encoder and decoder: the first pop
                # returns the tensor just pushed (bottleneck ++ itself), as in
                # the reference (nlt.py:180, 184-190)
                if query_featmaps:
                    query_x = query_x + query_featmaps.pop()
                query_y = layer_query.forward_segs(query_x, tape)
                query_x = [Seg(query_y)]
        return query_y

    # ------------------------------------------------------------------
    # loss / backward
    # ------------------------------------------------------------------
    def set_loss_grad_scale(self, scale):
        """1/global_bs of tf.nn.compute_average_loss (trainvali.py:277-278)."""
        self._loss_grad_scale = scale

    def compute_loss(self, pred, gt, **kwargs):
        loss = 0
        d_pred = None
        for weight, loss_func in self.wloss:
            if self._tape is not None:
                loss_func.grad_scale = (self._loss_grad_scale or 1.0) * weight
            else:
                loss_func.grad_scale = None
            loss += weight * loss_func(gt, pred, **kwargs)
            if self._tape is not None:
                d_pred = loss_func.d_pred if d_pred is None else d_pred + loss_func.d_pred
        self._d_pred = d_pred
        return loss

    def backward(self):
        """Fills .gradients (== d(sum_b loss_b * loss_grad_scale)/d(vars))."""
        if self._tape is None:
            raise RuntimeError('backward() needs a preceding call(..., mode="train")')
        self._tape.backward()
        self._tape = None
        self._d_pred = None

    # ------------------------------------------------------------------
    # visualisation (host side; SURVEY.md 8f row N4)
    # ------------------------------------------------------------------
    @staticmethod
    def psnr(im1, im2):
        """xiuminglib.metric.PSNR semantics (metric.py:105-151): luma, drange 1."""
        w = np.array([0.2126, 0.7152, 0.0722])
        a = np.clip(np.asarray(im1, dtype=np.float64), 0, 1) @ w
        b = np.clip(np.asarray(im2, dtype=np.float64), 0, 1) @ w
        mse = np.mean((a - b) ** 2)
        return float(10 * np.log10(1.0 / mse)) if mse > 0 else float('inf')

    @staticmethod
    def _linear2srgb(im):
        """IEC 61966-2-1 transfer curve on values in [0, 1] (xiuminglib img.linear2srgb)."""
        im = np.asarray(im, dtype=np.float64)
        return np.where(im <= 0.0031308, 12.92 * im, 1.055 * np.power(np.maximum(im, 0.0031308), 1 / 2.4) - 0.055)

    @staticmethod
    def _write_png(arr_0to1, path):
        """float [0, 1] -> uint8 by truncation (xiuminglib io.img.write_arr: `(arr * 255).astype(uint8)`) -> PNG."""
        from PIL import Image
        img = (np.asarray(arr_0to1) * 255).astype(np.uint8)
        Image.fromarray(img).save(path)
        return img

    def vis_batch(self, data_dict, outdir, mode, dump_raw_to=None, **_):
        """Per example i of the batch (nlt/models/nlt.py:207-271): `<i>_{base,pred,nn,gt}.png` (clipped to [0, 1],
        linear -> sRGB when the config says `linear_space`), `<i>_base-vs-pred.apng` / `<i>_gt-vs-pred.apng` flip
        books (unlabelled: the reference draws captions with xiuminglib), `<i>_metadata.json` with the ids and
        the luma PSNRs of prediction and diffuse base against the ground truth; `dump_raw_to` pickles the raw
        dictionary.  Everything here runs on the host after the tensors left the GPU."""
        import pickle
        from PIL import Image
        self._validate_mode(mode)
        os.makedirs(outdir, exist_ok=True)
        def to_np(t):
            a = t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
            return a.astype(np.float32) / 255 if a.dtype == np.uint8 else a       # uint8_inputs batches
        dec = lambda x: x.decode() if isinstance(x, bytes) else str(x)
        ids = [dec(x) for x in data_dict['id']]
        nn_ids = [dec(x) for x in data_dict['nn_id']]
        preds, bases = to_np(data_dict['pred_camspc']), to_np(data_dict['base_camspc'])
        nns = to_np(data_dict['nn_camspc']) if 'nn_camspc' in data_dict else None
        gts = None if mode == 'test' else to_np(data_dict['gt_camspc'])
        is_linear = self.config.getboolean('DEFAULT', 'linear_space', fallback=False)
        shown = (lambda x: self._linear2srgb(x)) if is_linear else (lambda x: x)
        for i, id_ in enumerate(ids):
            pred, base = np.clip(preds[i], 0, 1), np.clip(bases[i], 0, 1)
            gt = None if gts is None else np.clip(gts[i], 0, 1)
            frames = {'base': self._write_png(shown(base), os.path.join(outdir, '%d_base.png' % i)),
                      'pred': self._write_png(shown(pred), os.path.join(outdir, '%d_pred.png' % i))}
            if nns is not None:
                self._write_png(shown(np.clip(nns[i], 0, 1)), os.path.join(outdir, '%d_nn.png' % i))
            if gt is not None:
                frames['gt'] = self._write_png(shown(gt), os.path.join(outdir, '%d_gt.png' % i))
            for first, second in (('base', 'pred'), ('gt', 'pred')):
                if first in frames:
                    a, b = Image.fromarray(frames[first]), Image.fromarray(frames[second])
                    a.save(os.path.join(outdir, '%d_%s-vs-%s.apng' % (i, first, second)), format='PNG',
                           save_all=True, append_images=[b], duration=500, loop=0)
            meta = {'id': id_, 'nn_id': nn_ids[i]}
            if gt is not None:
                meta['pred_psnr'] = self.psnr(gt, pred)
                meta['base_psnr'] = self.psnr(gt, base)
            with open(os.path.join(outdir, '%d_metadata.json' % i), 'w') as h:
                json.dump(meta, h)
        if dump_raw_to is not None:
            raw = {k: (to_np(v) if torch.is_tensor(v) else v) for k, v in data_dict.items()}
            with open(dump_raw_to, 'wb') as h:
                pickle.dump(raw, h)

    def compile_batch_vis(self, batch_vis_dirs, outpref, mode, fps=6, **_):
        """train / vali: one HTML page with a row per visualised example (flip books + PSNRs); the reference also
        renders test batches into an MP4, which needs an encoder that is not part of this repo."""
        self._validate_mode(mode)
        if mode == 'test':
            raise NotImplementedError('MP4 compilation of test batches needs a video encoder (SURVEY.md 8f N4)')
        rows = []
        for d in batch_vis_dirs:
            for name in sorted(f for f in os.listdir(d) if f.endswith('_metadata.json')):
                i = name.split('_')[0]
                with open(os.path.join(d, name)) as h:
                    meta = json.load(h)
                cells = ['<td>%s</td>' % meta['id']]
                for pair in ('gt-vs-pred', 'base-vs-pred'):
                    f = os.path.join(d, '%s_%s.apng' % (i, pair))
                    cells.append('<td><img src="%s"></td>' % os.path.relpath(f, os.path.dirname(outpref) or '.')
                                 if os.path.exists(f) else '<td></td>')
                cells.append('<td>%s</td>' % ', '.join('%s %.2f dB' % (k, meta[k]) for k in ('pred_psnr', 'base_psnr')
                                                         if k in meta))
                rows.append('<tr>%s</tr>' % ''.join(cells))
        outpath = outpref + '.html'
        with open(outpath, 'w') as h:
            h.write('<html><head><title>NLT (%s)</title></head><body><table>\n%s\n</table></body></html>\n'
                    % (mode, '\n'.join(rows)))
        return outpath
