"""Res2Net mirror (reference: mvector/models/res2net.py:89-174), lowered.

  stem      7x7 stride-3 conv2d on the one-channel feature map (CONV_C1, BN folded, ReLU) -> 3x3 stride-2 max pool (POOL2D)
  Bottle2neck (res2net.py:10-86) on channel-last [B, T, F, C] maps:
      conv1 1x1 (BN folded, ReLU) -> split into `scale` groups of `width` channels
      groups 0 .. scale-2: 3x3 conv (stride s) + BN + ReLU; in 'normal' blocks group j adds the previous group's output
                            to its input (CONV gather ADD), in 'stage' blocks (first of a layer) every group is independent
      last group: passed through ('normal': EW copy) or 3x3 average pooled with stride s ('stage': POOL2D)
      all written into their slots of the concat buffer; conv3 1x1 + BN + residual (+ 1x1 stride-s downsample) + ReLU
  head      free (f, c) flatten -> pooling (ASP/SAP/TAP/TSP) -> bn2 -> linear -> bn3 folded into one product
"""
import math
from collections import OrderedDict

from .. import _lib as L
from ..engine import View
from .base import Backbone, bn_names
from .conv2d_util import fc_perm, lower_stem_c1, out_len, pack_conv_bn
from .pooling import check_pooling_type, head_shapes, lower_head, pack_head


class Res2Net(Backbone):
    def __init__(self, input_size, m_channels=32, layers=[3, 4, 6, 3], base_width=32, scale=2, embd_dim=192,
                 pooling_type='ASP'):
        super().__init__()
        check_pooling_type(pooling_type)
        if scale < 2:
            raise NotImplementedError('Res2Net: scale == 1 is not lowered')
        self.pooling_type = pooling_type
        self.input_size, self.embd_dim = input_size, embd_dim
        self.m, self.layers, self.base_width, self.scale = m_channels, list(layers), base_width, scale
        self.cat = m_channels * 8 * 4 * (input_size // base_width)

    def _blocks(self):
        inpl = self.m
        for li, nb in enumerate(self.layers, start=1):
            planes = self.m * (2 ** (li - 1))
            stride = 1 if li == 1 else 2
            for b in range(nb):
                first = b == 0
                ds = first and (stride != 1 or inpl != planes * 4)
                width = int(math.floor(planes * (self.base_width / 64.0)))
                yield f'layer{li}.{b}', inpl, planes, width, (stride if first else 1), first, ds
                inpl = planes * 4

    def param_shapes(self):
        d = OrderedDict()
        d['conv1.weight'] = (self.m, 1, 7, 7)
        bn_names(d, 'bn1', self.m)
        nums = self.scale - 1
        for p, inpl, planes, w, stride, stage, ds in self._blocks():
            d[p + '.conv1.weight'] = (w * self.scale, inpl, 1, 1)
            bn_names(d, p + '.bn1', w * self.scale)
            for j in range(nums):
                d[f'{p}.convs.{j}.weight'] = (w, w, 3, 3)
            for j in range(nums):
                bn_names(d, f'{p}.bns.{j}', w)
            d[p + '.conv3.weight'] = (planes * 4, w * self.scale, 1, 1)
            bn_names(d, p + '.bn3', planes * 4)
            if ds:
                d[p + '.downsample.0.weight'] = (planes * 4, inpl, 1, 1)
                bn_names(d, p + '.downsample.1', planes * 4)
        head_shapes(d, self.pooling_type, self.cat, self.embd_dim, 'bn2', 'linear', 'bn3')
        return d

    def _pack(self, sd, arena):
        o = self._off
        pack_conv_bn(sd, arena, o, 'stem', 'conv1.weight', 'bn1')
        for p, inpl, planes, w, stride, stage, ds in self._blocks():
            pack_conv_bn(sd, arena, o, p + '.c1', p + '.conv1.weight', p + '.bn1')
            for j in range(self.scale - 1):
                pack_conv_bn(sd, arena, o, f'{p}.k{j}', f'{p}.convs.{j}.weight', f'{p}.bns.{j}')
            pack_conv_bn(sd, arena, o, p + '.c3', p + '.conv3.weight', p + '.bn3')
            if ds:
                pack_conv_bn(sd, arena, o, p + '.ds', p + '.downsample.0.weight', p + '.downsample.1')
        C4 = self.m * 8 * 4
        o['head'] = pack_head(sd, arena, self.pooling_type, self.cat, 'bn2', 'linear', 'bn3',
                              perm=fc_perm(self.cat // C4, C4))

    def _lower(self, pb, B, T):
        o, sc = self._off, self.scale
        F = self.input_size
        s0, t, f = lower_stem_c1(pb, o['stem'], B, T, F, self.m, k=7, stride=3)
        tp, fp = out_len(t, 3, 2, 1), out_len(f, 3, 2, 1)
        x = pb.alloc(B * tp * fp, self.m)
        pb.pool2d(s0, x, L.POOL_MAX, t, f, tp, fp, k=3, stride=2, pad=1)
        pb.free(s0)
        t, f = tp, fp
        for p, inpl, planes, w, stride, stage, ds in self._blocks():
            to, fo = out_len(t, 3, stride, 1), out_len(f, 3, stride, 1)
            rows_in, rows_out = B * t * f, B * to * fo
            h = pb.alloc(rows_in, w * sc)
            pb.conv(x, h, o[p + '.c1']['w'], inpl, t, t, Fin=f, Fout=f, bias=o[p + '.c1']['b'], act=L.ACT_RELU)
            cat = pb.alloc(rows_out, w * sc)
            for j in range(sc - 1):
                e = o[f'{p}.k{j}']
                add_prev = (j > 0) and not stage
                pb.conv(h.cols(j * w, w), cat.cols(j * w, w), e['w'], 9 * w, t, to, Fin=f, Fout=fo, KT=3, KF=3, sT=stride,
                        sF=stride, padT=1, padF=1, bias=e['b'], act=L.ACT_RELU,
                        src2=cat.cols((j - 1) * w, w) if add_prev else None,
                        src2_mode=L.SRC2_ADD if add_prev else L.SRC2_NONE)
            last = h.cols((sc - 1) * w, w)
            if stage:
                pb.pool2d(last, cat.cols((sc - 1) * w, w), L.POOL_AVG, t, f, to, fo, k=3, stride=stride, pad=1)
            else:
                pb.ew(L.EW_COPY, last, cat.cols((sc - 1) * w, w), to * fo)
            pb.free(h)
            cout = planes * 4
            if ds:
                res = pb.alloc(rows_out, cout)
                pb.conv(x, res, o[p + '.ds']['w'], inpl, t, to, Fin=f, Fout=fo, sT=stride, sF=stride, bias=o[p + '.ds']['b'])
            else:
                res = x
            y = pb.alloc(rows_out, cout)
            pb.conv(cat, y, o[p + '.c3']['w'], w * sc, to, to, Fin=fo, Fout=fo, bias=o[p + '.c3']['b'], res=res,
                    act2=L.ACT_RELU)
            pb.free(cat)
            if ds:
                pb.free(res)
            pb.free(x)
            x, t, f = y, to, fo
        C4 = self.m * 8 * 4
        if f * C4 != self.cat:
            raise ValueError(f'input_size {F}: the flattened map has {f * C4} channels but the head was built for '
                             f'{self.cat} = m_channels*32*(input_size // base_width) (res2net.py:111)')
        lower_head(pb, o['head'], self.pooling_type, View(x.off, f * C4, 0, f * C4), B, t, self.embd_dim)
