"""Host logic and ABI surface.  CPU only (no kernels are launched)."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gen_feat_n_matches_reference_goldens():
    import numpy as np
    from util.net import gen_feat_n
    gold = np.load(os.path.join(ROOT, 'tests', 'golden', 'gen_feat_n_reference.npz'))
    for key in gold.files:
        a, b, f = (int(v) for v in key.split('_'))
        assert gen_feat_n(a, b, f) == gold[key].tolist(), key
    with pytest.raises(AssertionError):
        gen_feat_n(16, 8)


def test_network_structure_matches_reference_wiring():
    from networks import convnet
    net = convnet.Network(16, 256, 2, 2, norm_type='None', act_type='leakyrelu', pool_type='None')
    assert len(net.layers) == 14
    assert net.is_contracting == [True] * 7 + [False] * 7
    assert net.spatsize_changes == [1] + [0.5] * 6 + [2] * 6 + [1]
    kinds = [[(c.kind, c.k, c.s, c.cout, c.act) for c in blk.convs] for blk in net.layers]
    assert kinds[0] == [('conv', 1, 1, 16, None)]
    assert kinds[1] == [('conv', 2, 2, 16, 'leakyrelu'), ('conv', 2, 1, 16, 'leakyrelu')]
    assert kinds[6] == [('conv', 2, 2, 256, 'leakyrelu'), ('conv', 2, 1, 256, 'leakyrelu')]
    assert kinds[7] == [('deconv', 2, 2, 128, 'leakyrelu'), ('deconv', 2, 1, 128, 'leakyrelu')]
    assert kinds[13] == [('conv', 1, 1, 3, None)]
    sss = convnet.Network(16, 1024, 2, 2, norm_type='None', act_type='relu', pool_type='None')
    assert len(sss.layers) == 18
    with pytest.raises(AssertionError):
        convnet.Network(16, 256, 2, 2, norm_type=None)          # str2none asserts on non-strings
    # norm = pixel / instance: conv -> norm -> act, the activation moves into the norm op (convnet.py:50-59)
    for kind in ('pixel', 'instance'):
        nn_ = convnet.Network(16, 256, 2, 2, norm_type=kind, act_type='leakyrelu', pool_type='None')
        blk = nn_.layers[3]
        assert [c.act for c in blk.convs] == [None, None]
        assert [(n.kind, n.act, n.has_params) for n in blk.norms] == [(kind, 'leakyrelu', kind == 'instance')] * 2
        assert nn_.layers[0].norms == [None] and nn_.layers[13].norms == [None]     # bare 1x1 convs (:44, :85)
    for bad in (dict(norm_type='batch'), dict(norm_type='layer'), dict(pool_type='max'), dict(act_type='gelu')):
        kw = dict(norm_type='None', act_type='relu', pool_type='None')
        kw.update(bad)
        with pytest.raises(NotImplementedError):
            convnet.Network(16, 256, 2, 2, **kw)


def test_loss_string_grammar():
    from models.base import Model
    p = Model._parse_loss_and_weight
    assert p('1e+0lpips') == ('lpips', 1.0)
    assert p('barron') == ('barron', 1.0)
    assert p('10l2') == ('l2', 10.0)
    assert p('1e+2l1') == ('l1', 100.0)
    assert p('.5ssim') == ('ssim', 0.5)


def test_model_registry_and_config_keys():
    import models
    from util import io as ioutil
    Model = models.get_model_class('nlt')
    for name in ('dragon_specular.ini', 'dragon_sss.ini'):
        cfg = ioutil.read_config(name)
        m = Model(cfg)
        m.register_trainable()
        assert m.trainable_registered and m.trainable_variables == []
        assert len(m.net['query'].layers) == (14 if 'specular' in name else 18)
    cfg = ioutil.make_config(loss='barron,1e+0lpips')
    with pytest.raises(NotImplementedError):
        Model(cfg)                                   # N1: not on the accelerated path yet
    with pytest.raises(NotImplementedError):
        Model(ioutil.make_config(loss='nope'))


def test_no_cpu_fallback():
    import models
    from util import io as ioutil, synth
    if torch.cuda.is_available():
        pytest.skip('CUDA present')
    m = models.get_model_class('nlt')(ioutil.make_config(uvh=64, uvw=64, imh=64, imw=64))
    m.register_trainable()
    import nlt_native as nat
    with pytest.raises(nat.NativeError):
        m(synth.make_batch(1, 64, 64), mode='test')


def test_same_pad():
    from engine import same_pad
    assert same_pad(8, 2, 1) == (0, 1) and same_pad(8, 2, 2) == (0, 0) and same_pad(8, 3, 2) == (0, 1)
    assert same_pad(7, 3, 2) == (1, 1) and same_pad(8, 3, 1) == (1, 1)


def test_abi_library_loads_and_exports_every_declared_symbol():
    import nlt_native as nat
    hdr = open(os.path.join(ROOT, 'include', 'nlt_b200.h')).read()
    hdr = re.sub(r'/\*.*?\*/', '', hdr, flags=re.S)
    declared = set(re.findall(r'\b(nlt_[a-z0-9_]+)\s*\(', hdr))
    assert declared, 'no declarations parsed'
    assert declared == set(nat.exported_symbols())
    lib = nat.lib()          # loads the .so, binds every symbol (AttributeError if one is missing)
    raw = ctypes.CDLL(nat.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), name
    assert b'sm_90a' in lib.nlt_version()
    # argument validation happens before any CUDA call
    d = nat.GConvDesc()
    assert lib.nlt_gconv_fwd(ctypes.byref(d), None, 0, 0.0, None, 0, None, None) == -1
    assert lib.nlt_gconv_wgrad_workspace_bytes(ctypes.byref(d)) == -1
    assert lib.nlt_l2_loss_workspace_bytes(4, 1000) > 0
    assert lib.nlt_uv2cam_fwd(None, None, None, None, 1, 1, 1, 1, 1, 1, None, None, None, None, None, None) == -1


def test_desc_struct_layout_matches_header():
    """ctypes mirror == C struct: compile a probe that prints sizeof/offsetof."""
    import nlt_native as nat
    src = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "nlt_b200.h"
    int main(void) {
      printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(nlt_gconv_desc), offsetof(nlt_gconv_desc, seg_ptr),
             offsetof(nlt_gconv_desc, seg_sub), offsetof(nlt_gconv_desc, seg_C), offsetof(nlt_gconv_desc, Cout),
             offsetof(nlt_gconv_desc, w), offsetof(nlt_gconv_desc, w_n_stride));
      return 0; }'''
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        open(os.path.join(td, 'p.c'), 'w').write(src)
        subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), os.path.join(td, 'p.c'), '-o',
                               os.path.join(td, 'p')])
        out = subprocess.check_output([os.path.join(td, 'p')]).split()
    D = nat.GConvDesc
    want = [ctypes.sizeof(D), D.seg_ptr.offset, D.seg_sub.offset, D.seg_C.offset, D.Cout.offset, D.w.offset,
            D.w_n_stride.offset]
    assert [int(x) for x in out] == want


def test_synth_batch_properties():
    from util import synth
    b = synth.make_batch(2, 32, 32, seed=3, c_extra=4)
    assert b[1].shape == (2, 32, 32, 3) and b[2].shape == (2, 32, 32, 5) and b[4].shape == (2, 32, 32, 2)
    assert torch.equal(torch.round(b[1] * 255) / 255, b[1])
    frac_bg = float(((b[4] == 0).all(dim=3)).float().mean())
    assert 0.15 < frac_bg < 0.6
    assert torch.equal(b[4], b[4].half().float())


# ---- gradient bookkeeping of the tape (engine.contribute): first writer beta = 0, later ones beta = 1, ----
# ---- mask on the last; a small pointwise first contribution is parked and rides on the next launch     ----
class _Rec:
    """write_fn stand-in that records how it was called instead of launching a kernel."""

    def __init__(self, log, name):
        self.log, self.name = log, name

    def __call__(self, out, beta, mask, mask_act, term):
        self.log.append((self.name, beta, mask is not None, mask_act, term))


def _act(n_cons, act='leakyrelu'):
    import engine
    a = engine.Act(torch.zeros(1, 2, 2, 4), act=act, needs_grad=True)
    a.n_cons = n_cons
    return a


def test_contribute_plain_order_beta_and_mask():
    import engine
    log = []
    a = _act(3)
    for name in 'xyz':
        engine.contribute(a, _Rec(log, name))
    leaky = engine.nat.ACT_CODES['leakyrelu']
    assert log == [('x', 0.0, False, 0, None), ('y', 1.0, False, 0, None), ('z', 1.0, True, leaky, None)]
    assert a.grad is not None and a.n_contrib == 3


def test_contribute_parks_pointwise_first_contribution_and_fuses_it():
    import engine
    assert engine.FUSE_POINTWISE_DGRAD
    log = []
    a = _act(2)
    term = object()
    engine.contribute(a, _Rec(log, 'final1x1'), offer=(term, ()))
    assert log == [] and a.grad is None and a.pending is not None and a.n_contrib == 1
    engine.contribute(a, _Rec(log, 'down'), can_fuse=lambda t, out, mask: t is term and mask is not None)
    leaky = engine.nat.ACT_CODES['leakyrelu']
    # ONE launch: beta 0 (nothing was written before), mask (it is the last contribution), term attached
    assert log == [('down', 0.0, True, leaky, term)]
    assert a.pending is None and a.n_contrib == 2
    engine._PARKED.clear()


def test_contribute_parked_contribution_is_issued_alone_when_next_cannot_fuse():
    import engine
    log = []
    a = _act(3, act=None)
    engine.contribute(a, _Rec(log, 'final1x1'), offer=(object(), ()))
    engine.contribute(a, _Rec(log, 'tiled'), can_fuse=lambda t, out, mask: False)
    engine.contribute(a, _Rec(log, 'last'))
    assert log == [('final1x1', 0.0, False, 0, None), ('tiled', 1.0, False, 0, None), ('last', 1.0, False, 0, None)]
    engine._PARKED.clear()


def test_contribute_does_not_park_a_sole_or_late_contribution():
    import engine
    log = []
    a = _act(1)
    engine.contribute(a, _Rec(log, 'only'), offer=(object(), ()))
    assert [e[0] for e in log] == ['only'] and a.pending is None      # sole consumer: launched, masked
    b = _act(2)
    engine.contribute(b, _Rec(log, 'first'))
    engine.contribute(b, _Rec(log, 'second'), offer=(object(), ()))    # not first: plain accumulate
    assert log[-1][:3] == ('second', 1.0, True) and b.pending is None


def test_parked_contribution_without_follower_is_settled_by_the_tape():
    import engine
    log = []
    a = _act(2)
    tape = engine.Tape()
    tape.record(lambda: engine.contribute(a, _Rec(log, 'final1x1'), offer=(object(), ())))
    old = engine.USE_SIDE_STREAM
    engine.USE_SIDE_STREAM = False
    try:
        tape.backward()
    finally:
        engine.USE_SIDE_STREAM = old
    # the second consumer never contributed (its own gradient was None): the parked one must not be lost
    assert log == [('final1x1', 0.0, False, 0, None)] and a.grad is not None and a.pending is None


def test_vis_batch_outputs_and_psnr(tmp_path):
    """Host-side visualisation (SURVEY 8f N4; nlt/models/nlt.py:207-286): PNGs by truncating uint8 conversion,
    flip-book APNGs, metadata with luma PSNRs, optional raw pickle, HTML index."""
    import json
    import pickle
    import numpy as np
    from PIL import Image
    import models
    from util import io as ioutil
    m = models.get_model_class('nlt')(ioutil.read_config('dragon_specular.ini'))
    g = torch.Generator().manual_seed(3)
    B, H, W = 2, 6, 5
    gt = torch.rand(B, H, W, 3, generator=g)
    pred = (gt + 0.05 * torch.randn(B, H, W, 3, generator=g))            # leaves [0, 1]: must be clipped
    base = torch.rand(B, H, W, 3, generator=g)
    d = {'id': [b'trainvali_000000000_c_l', b'trainvali_000000001_c_l'], 'nn_id': [b'n0', b'n1'],
         'pred_camspc': pred, 'base_camspc': base, 'nn_camspc': base * 0.5, 'gt_camspc': gt}
    out = str(tmp_path / 'vis' / 'batch0')
    raw = str(tmp_path / 'raw.pkl')
    m.vis_batch(d, out, 'vali', dump_raw_to=raw)
    for i in range(B):
        for name in ('base', 'pred', 'nn', 'gt'):
            assert os.path.exists(os.path.join(out, '%d_%s.png' % (i, name)))
        got = np.array(Image.open(os.path.join(out, '%d_pred.png' % i)))
        want = (np.clip(pred[i].numpy(), 0, 1) * 255).astype(np.uint8)   # truncation, not rounding
        np.testing.assert_array_equal(got, want)
        ap = Image.open(os.path.join(out, '%d_gt-vs-pred.apng' % i))
        assert getattr(ap, 'n_frames', 1) == 2
        meta = json.load(open(os.path.join(out, '%d_metadata.json' % i)))
        assert meta['id'] == d['id'][i].decode() and meta['nn_id'] == d['nn_id'][i].decode()
        # luma PSNR, dynamic range 1, on the clipped images
        w = np.array([0.2126, 0.7152, 0.0722])
        a, b = np.clip(gt[i].numpy().astype(np.float64), 0, 1) @ w, np.clip(pred[i].numpy().astype(np.float64), 0, 1) @ w
        assert abs(meta['pred_psnr'] - 10 * np.log10(1.0 / np.mean((a - b) ** 2))) <= 1e-9
        assert meta['base_psnr'] < meta['pred_psnr']
    dumped = pickle.load(open(raw, 'rb'))
    np.testing.assert_array_equal(dumped['pred_camspc'], pred.numpy())
    page = m.compile_batch_vis([out], str(tmp_path / 'vis' / 'index'), 'vali')
    html = open(page).read()
    assert page.endswith('.html') and html.count('<tr>') == B and 'batch0/0_gt-vs-pred.apng' in html
    # test mode: no ground truth, no PSNRs; MP4 compilation is not offered
    out_t = str(tmp_path / 'vis' / 'test0')
    m.vis_batch({k: v for k, v in d.items() if k != 'gt_camspc'}, out_t, 'test')
    meta = json.load(open(os.path.join(out_t, '0_metadata.json')))
    assert 'pred_psnr' not in meta and not os.path.exists(os.path.join(out_t, '0_gt.png'))
    with pytest.raises(NotImplementedError):
        m.compile_batch_vis([out_t], str(tmp_path / 'vis' / 'video'), 'test')
    with pytest.raises(ValueError):
        m.vis_batch(d, out, 'predict')
    # linear -> sRGB transfer curve
    lin = np.array([0.0, 0.0031308, 0.5, 1.0])
    np.testing.assert_allclose(m._linear2srgb(lin), [0.0, 12.92 * 0.0031308, 1.055 * 0.5 ** (1 / 2.4) - 0.055, 1.0],
                               rtol=1e-12)


def test_barron_entry_point_host_side_and_gating(monkeypatch):
    """The workspace query of nlt_barron_loss is pure host code; losses.Barron constructs without a GPU."""
    import nlt_native as nat
    import losses
    lib = nat.lib()
    assert lib.nlt_barron_loss_workspace_bytes(1, 8, 8, 5) < 0           # 8 x 8 supports at most 3 levels
    assert lib.nlt_barron_loss_workspace_bytes(2, 64, 48, 5) > 4 * 2 * 3 * 64 * 48 * 2
    assert lib.nlt_barron_loss_workspace_bytes(0, 64, 64, 5) < 0
    b = losses.Barron(64, 48)
    assert (b.imw, b.imh) == (64, 48) and abs(b.LOG_Z_ALPHA1 - 1.185495232349193) < 1e-12


def test_opbench_layer_table_matches_the_network_wiring():
    """tools/opbench.py replays the two-stream wiring (SURVEY 8a table): 39 convs, concat widths 1024 / 640 / ... / 36."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('opbench', os.path.join(ROOT, 'tools', 'opbench.py'))
    ob = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ob)
    rows = {r[0]: r for r in ob.layer_table(uv=512, batch=1)}
    assert len(rows) == 39
    cin = {name: sum(r[5]) for name, r in rows.items()}
    assert [cin['query.%d.0' % i] for i in range(7, 14)] == [1024, 640, 320, 160, 80, 40, 36]
    assert cin['query.1.0'] == 32 and cin['obs.1.0'] == 16 and cin['query.6.0'] == 512
    assert rows['query.7.0'][4] == 8 and rows['query.13.0'][4] == 512 and rows['query.13.0'][6] == 3


def test_pack_arena_bump_allocation_and_rewind():
    """engine.PackArena: 256-byte aligned float32 views out of kept chunks, rewound (same addresses) at step begin;
    a request larger than a chunk gets its own chunk."""
    import torch
    import engine
    a = engine.PackArena()
    a.CHUNK = 4096
    dev = torch.device('cpu')
    x = a.alloc(1000, dev)
    y = a.alloc(300, dev)
    assert x.dtype == torch.float32 and x.numel() * 4 >= 1000 and y.numel() * 4 >= 300
    assert y.data_ptr() - x.data_ptr() == 1024 and (y.data_ptr() - x.data_ptr()) % 256 == 0
    big = a.alloc(3 * 4096, dev)                     # does not fit the first chunk: a chunk of its own
    assert big.numel() * 4 >= 3 * 4096 and len(a.chunks) == 2
    z = a.alloc(3000, dev)                           # fits neither what is left of chunk 0 nor chunk 1
    assert len(a.chunks) == 3 and z.numel() * 4 >= 3000
    a.reset()
    assert a.alloc(1000, dev).data_ptr() == x.data_ptr()      # a captured graph may keep the addresses
    assert a.alloc(300, dev).data_ptr() == y.data_ptr()


def test_scheduling_switches_have_the_documented_defaults():
    """NLT_SIDE_STREAMS = 2 weight-gradient streams, NLT_PACK_AHEAD off, side stream on (DESIGN.md 4.1); read in a fresh
    interpreter so that this process's engine module is left alone."""
    import os
    import subprocess
    import sys
    import engine
    env = {k: v for k, v in os.environ.items() if k not in ('NLT_SIDE_STREAMS', 'NLT_PACK_AHEAD', 'NLT_NO_SIDE_STREAM')}
    pkg = os.path.dirname(os.path.abspath(engine.__file__))
    out = subprocess.run([sys.executable, '-c',
                          'import sys; sys.path.insert(0, %r); import engine as e; '
                          'print(e.N_SIDE_STREAMS, e.PACK_AHEAD, e.USE_SIDE_STREAM)' % pkg],
                         env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert out.stdout.split() == ['2', 'False', 'True']
    ws = engine.Workspace()
    assert ws.sub(0) is ws and ws.sub(1) is ws.sub(1) and ws.sub(1) is not ws
