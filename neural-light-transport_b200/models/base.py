"""Model base class: loss-string parsing, layer registration, mode validation -- the parts of the reference's
`models.base.Model` protocol (nlt/models/base.py:26-140) that the drivers and `models.nlt` rely on.  No Keras
trackability here: parameters live in one flat bucket owned by the concrete model; `register_trainable()` still
publishes the `net_<name>_layer<i>` aliases, which are the reference's checkpoint key prefixes."""
import losses
from networks import base as basenet

_MODES = ('train', 'vali', 'test')

# loss name -> constructor (nlt/models/base.py:41-61; 'elpips' needs the TF-only E-LPIPS package and is not offered)
_LOSS_TABLE = {
    'l1': lambda: losses.L1(),
    'l2': lambda: losses.L2(),
    'ssim': lambda: losses.SSIM(1 - 0),
}


def _float_or_none(text):
    try:
        return float(text)
    except ValueError:
        return None


class Model:
    def __init__(self, config):
        self.config = config
        self.net = {'main': basenet.Network()}   # concrete models replace this with their named networks
        self.trainable_registered = False        # flipped by register_trainable(); the drivers assert on it
        self.wloss = self._init_loss()           # [(weight, loss object), ...] in config order

    # ---- 'loss = barron,1e+0lpips' style strings ----
    def _init_loss(self):
        pairs = []
        for item in self.config.get('DEFAULT', 'loss').split(','):
            name, weight = self._parse_loss_and_weight(item)
            if name == 'barron':     # needs the image size (nlt/models/nlt.py:78-79); experimental, see losses.Barron
                loss = losses.Barron(self.config.getint('DEFAULT', 'imw'), self.config.getint('DEFAULT', 'imh'))
            elif name == 'lpips':    # needs the reference's frozen graph, which is not shipped: see losses.LPIPS
                loss = losses.LPIPS(per_ch=False,
                                    weights_path=self.config.get('DEFAULT', losses.LPIPS.KEY, fallback=None))
            elif name in _LOSS_TABLE:
                loss = _LOSS_TABLE[name]()
            else:
                raise NotImplementedError(name)
            pairs.append((weight, loss))
        return pairs

    @staticmethod
    def _parse_loss_and_weight(weight_loss_str):
        """'1e+2lpips' -> ('lpips', 100.0); 'l2' -> ('l2', 1.0).  The weight is the LONGEST leading substring that
        `float()` accepts (nlt/models/base.py:63-77), so '1e+0lpips' reads 1e+0, not 1."""
        text = weight_loss_str
        cut = next((i for i in range(len(text), -1, -1) if _float_or_none(text[:i]) is not None), None)
        if cut is None:
            return text, 1.
        return text[cut:], float(text[:cut])

    # ---- layer aliases ----
    def register_trainable(self):
        """Publishes every layer of every network in `self.net` as attribute `net_<network>_layer<index>`
        (nlt/models/base.py:79-101: in the reference this is what makes Keras track the variables; here it keeps
        the attribute names -- and thereby checkpoint keys -- identical)."""
        aliases = {}
        for net_name, net in self.net.items():
            stem = 'net_' + net_name
            assert stem.isidentifier(), (
                "Prepending 'net_' to your network name '{net}' doesn't make a valid identifier; "
                "change your network name").format(net=net_name)
            for index, layer in enumerate(net.layers):
                alias = '%s_layer%d' % (stem, index)
                assert alias not in aliases and not hasattr(self, alias), \
                    "Can't register `%s` because it is already an attribute" % alias
                aliases[alias] = layer
        for alias, layer in aliases.items():
            setattr(self, alias, layer)
        self._registered = list(aliases)
        self.trainable_registered = True

    @staticmethod
    def _validate_mode(mode):
        if mode not in _MODES:
            raise ValueError(mode)

    # ---- protocol stubs ----
    def __call__(self, batch, mode=None, **kwargs):
        return self.call(batch, mode, **kwargs)

    def call(self, batch, mode):
        raise NotImplementedError

    def compute_loss(self, pred, gt, **kwargs):
        raise NotImplementedError

    def vis_batch(self, data_dict, outdir, mode, dump_raw_to=None):
        raise NotImplementedError

    def compile_batch_vis(self, batch_vis_dirs, outpref, mode):
        raise NotImplementedError
