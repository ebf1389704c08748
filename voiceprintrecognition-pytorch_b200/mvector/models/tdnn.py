"""TDNN (x-vector) mirror (reference: mvector/models/tdnn.py:9-68): five *valid* (unpadded) Conv1d layers, each
relu(conv) -> BN (tdnn.py:57-65; the 5th has no BN), ASP(512), bn5 -> linear -> bn6 folded into one product."""
from collections import OrderedDict

from .. import _lib as L
from .base import Backbone, bn_affine, bn_names, conv1d_weight
from .pooling import check_pooling_type, head_shapes, lower_head, pack_head

_KS = (5, 3, 3, 1, 1)
_DIL = (1, 2, 3, 1, 1)


class TDNN(Backbone):
    def __init__(self, input_size, channels=512, embd_dim=192, pooling_type='ASP'):
        super().__init__()
        check_pooling_type(pooling_type)
        self.pooling_type = pooling_type
        self.input_size, self.channels, self.embd_dim = input_size, channels, embd_dim

    def param_shapes(self):
        d = OrderedDict()
        c = self.channels
        for i, k in enumerate(_KS, start=1):
            d[f'td_layer{i}.weight'] = (c, self.input_size if i == 1 else c, k)
            d[f'td_layer{i}.bias'] = (c,)
            if i < 5:
                bn_names(d, f'bn{i}', c)
        head_shapes(d, self.pooling_type, c, self.embd_dim, 'bn5', 'linear', 'bn6')
        return d

    def _pack(self, sd, arena):
        o = self._off
        for i in range(1, 6):
            e = dict(w=arena.add_conv(f'td{i}.w', conv1d_weight(sd[f'td_layer{i}.weight'])),
                     b=arena.add(f'td{i}.b', sd[f'td_layer{i}.bias']))
            if i < 5:
                s, h = bn_affine(sd, f'bn{i}')
                e['s'], e['h'] = arena.add(f'bn{i}.s', s), arena.add(f'bn{i}.h', h)
            o[f'td{i}'] = e
        o['head'] = pack_head(sd, arena, self.pooling_type, self.channels, 'bn5', 'linear', 'bn6')

    def _lower(self, pb, B, T):
        o, c = self._off, self.channels
        x = pb.input_view1d(self.input_size, B * T, T)
        t = T
        for i, (k, dil) in enumerate(zip(_KS, _DIL), start=1):
            tout = t - dil * (k - 1)
            if tout < 1:
                raise ValueError(f'{T} frames is too short for the TDNN receptive field')
            e = o[f'td{i}']
            y = pb.alloc(B * tout, c)
            pb.conv(x, y, e['w'], k * x.C, t, tout, KT=k, dT=dil, bias=e['b'], act=L.ACT_RELU,
                    post=(e['s'], e['h']) if i < 5 else None)
            if x.off != L.BUF_INPUT:
                pb.free(x)
            x, t = y, tout
        lower_head(pb, o['head'], self.pooling_type, x, B, t, self.embd_dim)
