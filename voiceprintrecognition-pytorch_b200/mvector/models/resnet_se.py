"""ResNetSE mirror (reference: mvector/models/resnet_se.py:65-145), lowered.

SEBottleneck (resnet_se.py:23-44) on channel-last [B, T, F, C] maps:
  CONV 1x1 (BN folded, ReLU) -> CONV 3x3 stride s (BN folded, ReLU) -> CONV 1x1 (BN folded)
  -> COLSTATS mean over T*F -> two tiny CONVs (SE MLP, sigmoid) -> EW relu(out * gate + residual)
The final reshape to [B, C*F/8, T/8] is free in this layout; ASP / bn2 / linear / bn3 take (f, c)-permuted weights and
bn2 -> linear -> bn3 collapse into one product."""
from collections import OrderedDict

from .. import _lib as L
from ..engine import View
from .base import Backbone, bn_names
from .conv2d_util import fc_perm, lower_stem_c1, out_len, pack_conv_bn
from .pooling import check_pooling_type, head_shapes, lower_head, pack_head


class ResNetSE(Backbone):
    def __init__(self, input_size, layers=[3, 4, 6, 3], num_filters=[32, 64, 128, 256], embd_dim=192,
                 pooling_type='ASP'):
        super().__init__()
        check_pooling_type(pooling_type)
        self.pooling_type = pooling_type
        self.input_size, self.embd_dim = input_size, embd_dim
        self.layers, self.nf = list(layers), list(num_filters)
        self.F8 = input_size // 8
        self.cat = self.nf[3] * 2 * self.F8

    def _blocks(self):
        inpl = self.nf[0]
        for li, (nb, planes) in enumerate(zip(self.layers, self.nf), start=1):
            for b in range(nb):
                stride = 2 if (li > 1 and b == 0) else 1
                ds = b == 0 and (stride != 1 or inpl != planes * 2)
                yield f'layer{li}.{b}', inpl, planes, stride, ds
                inpl = planes * 2

    def param_shapes(self):
        d = OrderedDict()
        d['conv1.weight'] = (self.nf[0], 1, 3, 3)
        bn_names(d, 'bn1', self.nf[0])
        for p, inpl, planes, stride, ds in self._blocks():
            d[p + '.conv1.weight'] = (planes, inpl, 1, 1)
            bn_names(d, p + '.bn1', planes)
            d[p + '.conv2.weight'] = (planes, planes, 3, 3)
            bn_names(d, p + '.bn2', planes)
            d[p + '.conv3.weight'] = (planes * 2, planes, 1, 1)
            bn_names(d, p + '.bn3', planes * 2)
            d[p + '.se.fc.0.weight'] = (planes * 2 // 8, planes * 2)
            d[p + '.se.fc.0.bias'] = (planes * 2 // 8,)
            d[p + '.se.fc.2.weight'] = (planes * 2, planes * 2 // 8)
            d[p + '.se.fc.2.bias'] = (planes * 2,)
            if ds:
                d[p + '.downsample.0.weight'] = (planes * 2, inpl, 1, 1)
                bn_names(d, p + '.downsample.1', planes * 2)
        head_shapes(d, self.pooling_type, self.cat, self.embd_dim, 'bn2', 'linear', 'bn3')
        return d

    def _pack(self, sd, arena):
        o = self._off
        pack_conv_bn(sd, arena, o, 'stem', 'conv1.weight', 'bn1')
        for p, inpl, planes, stride, ds in self._blocks():
            pack_conv_bn(sd, arena, o, p + '.c1', p + '.conv1.weight', p + '.bn1')
            pack_conv_bn(sd, arena, o, p + '.c2', p + '.conv2.weight', p + '.bn2')
            pack_conv_bn(sd, arena, o, p + '.c3', p + '.conv3.weight', p + '.bn3')
            if ds:
                pack_conv_bn(sd, arena, o, p + '.ds', p + '.downsample.0.weight', p + '.downsample.1')
            o[p + '.se'] = dict(w1=arena.add(p + '.se.w1', sd[p + '.se.fc.0.weight']),
                                b1=arena.add(p + '.se.b1', sd[p + '.se.fc.0.bias']),
                                w2=arena.add(p + '.se.w2', sd[p + '.se.fc.2.weight']),
                                b2=arena.add(p + '.se.b2', sd[p + '.se.fc.2.bias']))
        o['head'] = pack_head(sd, arena, self.pooling_type, self.cat, 'bn2', 'linear', 'bn3',
                              perm=fc_perm(self.F8, self.nf[3] * 2))

    def _lower(self, pb, B, T):
        o = self._off
        x, t, f = lower_stem_c1(pb, o['stem'], B, T, self.input_size, self.nf[0])
        for p, inpl, planes, stride, ds in self._blocks():
            to, fo = out_len(t, 3, stride, 1), out_len(f, 3, stride, 1)
            h1 = pb.alloc(B * t * f, planes)
            pb.conv(x, h1, o[p + '.c1']['w'], inpl, t, t, Fin=f, Fout=f, bias=o[p + '.c1']['b'], act=L.ACT_RELU)
            h2 = pb.alloc(B * to * fo, planes)
            pb.conv(h1, h2, o[p + '.c2']['w'], 9 * planes, t, to, Fin=f, Fout=fo, KT=3, KF=3, sT=stride, sF=stride,
                    padT=1, padF=1, bias=o[p + '.c2']['b'], act=L.ACT_RELU)
            pb.free(h1)
            h3 = pb.alloc(B * to * fo, planes * 2)
            pb.conv(h2, h3, o[p + '.c3']['w'], planes, to, to, Fin=fo, Fout=fo, bias=o[p + '.c3']['b'])
            pb.free(h2)
            sq = pb.alloc(B, planes * 2)
            pb.colstats(h3, sq, to * fo, L.STATS_MEAN)
            se = o[p + '.se']
            g1 = pb.alloc(B, planes * 2 // 8)
            pb.conv(sq, g1, se['w1'], planes * 2, 1, 1, bias=se['b1'], act=L.ACT_RELU, engine=L.ENGINE_FFMA)
            g2 = pb.alloc(B, planes * 2)
            pb.conv(g1, g2, se['w2'], planes * 2 // 8, 1, 1, bias=se['b2'], act=L.ACT_SIGMOID, engine=L.ENGINE_FFMA)
            if ds:
                res = pb.alloc(B * to * fo, planes * 2)
                pb.conv(x, res, o[p + '.ds']['w'], inpl, t, to, Fin=f, Fout=fo, sT=stride, sF=stride,
                        bias=o[p + '.ds']['b'])
            else:
                res = x
            y = pb.alloc(B * to * fo, planes * 2)
            pb.ew(L.EW_GATE_RES, h3, y, to * fo, gate=g2, res=res, act2=L.ACT_RELU)
            if ds:
                pb.free(res)
            for v in (g2, g1, sq, h3, x):
                pb.free(v)
            x, t, f = y, to, fo
        assert f == self.F8, 'input_size must be a multiple of 8'
        C4 = self.nf[3] * 2
        lower_head(pb, o['head'], self.pooling_type, View(x.off, f * C4, 0, f * C4), B, t, self.embd_dim)
