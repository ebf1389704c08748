"""CAMPPlus mirror (reference: mvector/models/campplus.py:295-357), lowered.

  FCM head (campplus.py:257-292): five 3x3 conv2d stages on [B, T, F, 32] maps, BN folded into the conv weights
    (conv -> BN -> ReLU order), residual add + ReLU in the conv epilogue; freq stride 2 three times (F -> F/8).
  TDNNLayer (campplus.py:41-68): k5 stride-2 conv1d over the flattened (f, c) columns.
  CAMDenseTDNNLayer (campplus.py:114-150), 52 of them: BN-ReLU -> 1x1 -> BN-ReLU -> CAMLayer.  Lowered per layer to
    CONV(prologue = BN+ReLU on the dense-concat slice, BN2 folded, ReLU)  ->  COLSTATS(SEG_CONTEXT)  ->  two tiny
    CONVs (context MLP)  ->  CONV(k3 dilated local conv, epilogue multiplies the sigmoid gate, output written into
    its 32-column slot of the block's concat buffer -- no torch.cat).
  StatsPool (unbiased std) + DenseLayer with BN(affine=False) folded.
"""
import math
from collections import OrderedDict

from .. import _lib as L
from ..engine import View
from .base import Backbone, _np64, bn_affine, bn_names, conv1d_weight
from .conv2d_util import fc_perm, lower_stem_c1, out_len, pack_conv_bn

_BLOCKS = ((12, 3, 1), (24, 3, 2), (16, 3, 2))
_SEG = 100


class CAMPPlus(Backbone):
    def __init__(self, input_size, embd_dim=512, growth_rate=32, bn_size=4, init_channels=128,
                 config_str='batchnorm-relu', memory_efficient=True):
        super().__init__()
        if config_str != 'batchnorm-relu':
            raise NotImplementedError("CAMPPlus: only config_str='batchnorm-relu' is lowered")
        self.input_size, self.embd_dim = input_size, embd_dim
        self.growth, self.bn_ch, self.init_channels = growth_rate, bn_size * growth_rate, init_channels
        self.m = 32
        self.F8 = math.ceil(input_size / 8)

    def param_shapes(self):
        d = OrderedDict()
        m = self.m
        d['head.conv1.weight'] = (m, 1, 3, 3)
        bn_names(d, 'head.bn1', m)
        for layer in ('layer1', 'layer2'):
            for b in range(2):
                p = f'head.{layer}.{b}'
                d[p + '.conv1.weight'] = (m, m, 3, 3)
                bn_names(d, p + '.bn1', m)
                d[p + '.conv2.weight'] = (m, m, 3, 3)
                bn_names(d, p + '.bn2', m)
                if b == 0:
                    d[p + '.shortcut.0.weight'] = (m, m, 1, 1)
                    bn_names(d, p + '.shortcut.1', m)
        d['head.conv2.weight'] = (m, m, 3, 3)
        bn_names(d, 'head.bn2', m)
        ch = m * self.F8
        d['xvector.tdnn.linear.weight'] = (self.init_channels, ch, 5)
        bn_names(d, 'xvector.tdnn.nonlinear.batchnorm', self.init_channels)
        ch = self.init_channels
        for bi, (nl, k, dil) in enumerate(_BLOCKS, start=1):
            for li in range(nl):
                p = f'xvector.block{bi}.tdnnd{li + 1}'
                cin = ch + li * self.growth
                bn_names(d, p + '.nonlinear1.batchnorm', cin)
                d[p + '.linear1.weight'] = (self.bn_ch, cin, 1)
                bn_names(d, p + '.nonlinear2.batchnorm', self.bn_ch)
                d[p + '.cam_layer.linear_local.weight'] = (self.growth, self.bn_ch, k)
                d[p + '.cam_layer.linear1.weight'] = (self.bn_ch // 2, self.bn_ch, 1)
                d[p + '.cam_layer.linear1.bias'] = (self.bn_ch // 2,)
                d[p + '.cam_layer.linear2.weight'] = (self.growth, self.bn_ch // 2, 1)
                d[p + '.cam_layer.linear2.bias'] = (self.growth,)
            ch = ch + nl * self.growth
            bn_names(d, f'xvector.transit{bi}.nonlinear.batchnorm', ch)
            d[f'xvector.transit{bi}.linear.weight'] = (ch // 2, ch, 1)
            ch //= 2
        bn_names(d, 'xvector.out_nonlinear.batchnorm', ch)
        d['xvector.dense.linear.weight'] = (self.embd_dim, ch * 2, 1)
        bn_names(d, 'xvector.dense.nonlinear.batchnorm', self.embd_dim, affine=False)
        return d

    def _pack(self, sd, arena):
        o = self._off
        pack_conv_bn(sd, arena, o, 'stem', 'head.conv1.weight', 'head.bn1')
        for layer in ('layer1', 'layer2'):
            for bi in range(2):
                p = f'head.{layer}.{bi}'
                pack_conv_bn(sd, arena, o, p + '.c1', p + '.conv1.weight', p + '.bn1')
                pack_conv_bn(sd, arena, o, p + '.c2', p + '.conv2.weight', p + '.bn2')
                if bi == 0:
                    pack_conv_bn(sd, arena, o, p + '.sc', p + '.shortcut.0.weight', p + '.shortcut.1')
        pack_conv_bn(sd, arena, o, 'head.c2', 'head.conv2.weight', 'head.bn2')
        # TDNN layer: K columns (kt, f*32+c) <- reference channel c*F8+f
        perm = fc_perm(self.F8, self.m)
        Wt = _np64(sd['xvector.tdnn.linear.weight'])[:, perm, :]             # [N, mycol, kt]
        s, h = bn_affine(sd, 'xvector.tdnn.nonlinear.batchnorm')
        o['tdnn'] = dict(w=arena.add_conv('tdnn.w', conv1d_weight(Wt) * s[:, None]), b=arena.add('tdnn.b', h))
        for bi, (nl, k, dil) in enumerate(_BLOCKS, start=1):
            for li in range(nl):
                p = f'xvector.block{bi}.tdnnd{li + 1}'
                s1, h1 = bn_affine(sd, p + '.nonlinear1.batchnorm')
                s2, h2 = bn_affine(sd, p + '.nonlinear2.batchnorm')
                o[p] = dict(
                    pre_s=arena.add(p + '.pre_s', s1), pre_h=arena.add(p + '.pre_h', h1),
                    w1=arena.add_conv(p + '.w1', _np64(sd[p + '.linear1.weight'])[:, :, 0] * s2[:, None]),
                    b1=arena.add(p + '.b1', h2),
                    wl=arena.add_conv(p + '.wl', conv1d_weight(sd[p + '.cam_layer.linear_local.weight'])),
                    wa=arena.add(p + '.wa', _np64(sd[p + '.cam_layer.linear1.weight'])[:, :, 0]),
                    ba=arena.add(p + '.ba', sd[p + '.cam_layer.linear1.bias']),
                    wb=arena.add(p + '.wb', _np64(sd[p + '.cam_layer.linear2.weight'])[:, :, 0]),
                    bb=arena.add(p + '.bb', sd[p + '.cam_layer.linear2.bias']))
            p = f'xvector.transit{bi}'
            s, h = bn_affine(sd, p + '.nonlinear.batchnorm')
            o[p] = dict(pre_s=arena.add(p + '.pre_s', s), pre_h=arena.add(p + '.pre_h', h),
                        w=arena.add_conv(p + '.w', _np64(sd[p + '.linear.weight'])[:, :, 0]))
        s, h = bn_affine(sd, 'xvector.out_nonlinear.batchnorm')
        o['out_bn'] = (arena.add('out_bn.s', s), arena.add('out_bn.h', h))
        s, h = bn_affine(sd, 'xvector.dense.nonlinear.batchnorm')
        W = _np64(sd['xvector.dense.linear.weight'])[:, :, 0]
        o['dense'] = dict(w=arena.add('dense.w', W * s[:, None]), b=arena.add('dense.b', h))

    def _lower(self, pb, B, T):
        o, m = self._off, self.m
        # ---- FCM head ----
        x, _, f = lower_stem_c1(pb, o['stem'], B, T, self.input_size, m)
        for layer in ('layer1', 'layer2'):
            for bi in range(2):
                p = f'head.{layer}.{bi}'
                s = 2 if bi == 0 else 1
                fo = out_len(f, 3, s, 1)
                h = pb.alloc(B * T * fo, m)
                pb.conv(x, h, o[p + '.c1']['w'], 9 * m, T, T, Fin=f, Fout=fo, KT=3, KF=3, sF=s, padT=1, padF=1,
                        bias=o[p + '.c1']['b'], act=L.ACT_RELU)
                if bi == 0:
                    sc = pb.alloc(B * T * fo, m)
                    pb.conv(x, sc, o[p + '.sc']['w'], m, T, T, Fin=f, Fout=fo, sF=s, bias=o[p + '.sc']['b'])
                else:
                    sc = x
                y = pb.alloc(B * T * fo, m)
                pb.conv(h, y, o[p + '.c2']['w'], 9 * m, T, T, Fin=fo, Fout=fo, KT=3, KF=3, padT=1, padF=1,
                        bias=o[p + '.c2']['b'], res=sc, act2=L.ACT_RELU)
                pb.free(h)
                if bi == 0:
                    pb.free(sc)
                pb.free(x)
                x, f = y, fo
        fo = out_len(f, 3, 2, 1)
        assert fo == self.F8
        y = pb.alloc(B * T * fo, m)
        pb.conv(x, y, o['head.c2']['w'], 9 * m, T, T, Fin=f, Fout=fo, KT=3, KF=3, sF=2, padT=1, padF=1,
                bias=o['head.c2']['b'], act=L.ACT_RELU)
        pb.free(x)
        # ---- [B, T, F8, 32] viewed as [B*T, F8*32]; TDNN layer k5 stride 2 ----
        flat = View(y.off, fo * m, 0, fo * m)
        T2 = out_len(T, 5, 2, 2)
        ch = self.init_channels
        g = self.growth
        M = B * T2
        nseg = (T2 + _SEG - 1) // _SEG
        cat = pb.alloc(M, ch + _BLOCKS[0][0] * g)
        pb.conv(flat, cat.cols(0, ch), o['tdnn']['w'], 5 * fo * m, T, T2, KT=5, sT=2, padT=2, bias=o['tdnn']['b'],
                act=L.ACT_RELU)
        pb.free(y)
        for bi, (nl, k, dil) in enumerate(_BLOCKS, start=1):
            for li in range(nl):
                e = o[f'xvector.block{bi}.tdnnd{li + 1}']
                cin = ch + li * g
                hbuf = pb.alloc(M, self.bn_ch)
                pb.conv(cat.cols(0, cin), hbuf, e['w1'], cin, T2, T2, pre=(e['pre_s'], e['pre_h']), pre_relu=True,
                        bias=e['b1'], act=L.ACT_RELU)
                ctx = pb.alloc(B * nseg, self.bn_ch)
                pb.colstats(hbuf, ctx, T2, L.STATS_SEG_CONTEXT, seg_len=_SEG, n_seg=nseg)
                c1 = pb.alloc(B * nseg, self.bn_ch // 2)
                pb.conv(ctx, c1, e['wa'], self.bn_ch, 1, 1, bias=e['ba'], act=L.ACT_RELU, B=B * nseg,
                        engine=L.ENGINE_FFMA)
                gate = pb.alloc(B * nseg, g)
                pb.conv(c1, gate, e['wb'], self.bn_ch // 2, 1, 1, bias=e['bb'], act=L.ACT_SIGMOID, B=B * nseg,
                        engine=L.ENGINE_FFMA)
                pb.conv(hbuf, cat.cols(cin, g), e['wl'], k * self.bn_ch, T2, T2, KT=k, dT=dil, padT=(k - 1) // 2 * dil,
                        gate=gate, seg_len=_SEG, n_seg=nseg)
                for v in (gate, c1, ctx, hbuf):
                    pb.free(v)
            ch = ch + nl * g
            e = o[f'xvector.transit{bi}']
            last = bi == len(_BLOCKS)
            nxt = pb.alloc(M, ch // 2 + (0 if last else _BLOCKS[bi][0] * g))
            pb.conv(cat, nxt.cols(0, ch // 2), e['w'], ch, T2, T2, pre=(e['pre_s'], e['pre_h']), pre_relu=True,
                    post=o['out_bn'] if last else None, act2=L.ACT_RELU if last else L.ACT_NONE)
            pb.free(cat)
            cat, ch = nxt, ch // 2
        stats = pb.alloc(B, 2 * ch)
        pb.colstats(cat, stats, T2, L.STATS_MEAN_STD_UNBIASED)
        pb.free(cat)
        pb.conv(stats, pb.output_view(self.embd_dim, B), o['dense']['w'], 2 * ch, 1, 1, bias=o['dense']['b'],
                engine=L.ENGINE_FFMA)
