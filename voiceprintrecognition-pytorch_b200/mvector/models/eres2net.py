"""ERes2Net / ERes2NetV2 mirrors (reference: mvector/models/eres2net.py:173-263 and :383-456, two_emb_layer=False), lowered.

BasicBlockERes2Net(_diff_AFF) == BasicBlockERes2NetV2(_AFF) (eres2net.py:55-170, 266-381) on channel-last [B, T, F, C]
maps; activation is Hardtanh(0, 20) (eres2net.py:12-15) except the stem's plain ReLU (:243); every BN follows its conv and
is folded.
  conv1 1x1 (stride s)              CONV (+hardtanh)
  split into `scale` groups; group j: input = prev + x_j (CONV gather ADD) or AFF(prev, x_j) (eres2net.py:32-52):
     att = BN(conv(SiLU(BN(conv(cat(prev, x_j))))))   two CONVs (gather CONCAT, BN folded)   then EW AFF blend
     3x3 conv + BN + hardtanh -> written into its slot of the concat buffer
  conv3 1x1 + BN + shortcut + hardtanh              one CONV (residual + act2 in the epilogue)
ERes2Net:   bottom-up fusion of all four stages (:246-253): 3x3 stride-2 downsample CONVs + AFF; TSTP pooling; seg_1.
ERes2NetV2: only out3 -> layer3_ds -> fuse34 with out4 (:437-440).

Group widths that are not multiples of 4 (ERes2NetV2's default base_width 26 gives 13, 26, 52, 104) are zero-padded to
the next multiple of 4 at pack time: padded channels carry zero weights and zero bias, stay exactly 0 through
Hardtanh / SiLU / the AFF blend (x*(1+tanh 0) + y*(1-tanh 0) with x = y = 0), and meet zero columns in the next layer.
"""
import math
from collections import OrderedDict

import numpy as np

from .. import _lib as L
from ..engine import View
from .base import Backbone, _np64, bn_names
from .conv2d_util import conv2d_weight, fc_perm, fold_conv_bn, lower_stem_c1, out_len, pack_conv_bn

HT = L.ACT_HARDTANH20


def _pad4(n):
    return (n + 3) // 4 * 4


def _aff_names(d, p, channels, r=4):
    inter = int(channels // r)
    d[p + '.local_att.0.weight'] = (inter, channels * 2, 1, 1)
    d[p + '.local_att.0.bias'] = (inter,)
    bn_names(d, p + '.local_att.1', inter)
    d[p + '.local_att.3.weight'] = (channels, inter, 1, 1)
    d[p + '.local_att.3.bias'] = (channels,)
    bn_names(d, p + '.local_att.4', channels)


def _grp_rows(M, w, wp, g):
    """[g*w, ...] -> [g*wp, ...]: every group of w rows is followed by wp - w zero rows."""
    if w == wp:
        return M
    out = np.zeros((g * wp,) + M.shape[1:], dtype=M.dtype)
    for j in range(g):
        out[j * wp:j * wp + w] = M[j * w:(j + 1) * w]
    return out


def _grp_cols(M, w, wp, g):
    return _grp_rows(M.T, w, wp, g).T if w != wp else M


class ERes2Net(Backbone):
    # deep 2-D residual net: the tensor core's accumulate truncation adds up coherently through ~50 layers (the 55 M
    # variant at T = 998 measured 1.06e-4 with single accumulators up to K = 1536, 6.4e-5 with 256-element chunks)
    tc_chunk_policy = (512, 256)

    _BASE_WIDTH, _EXPANSION = 32, 2

    def __init__(self, input_size, block=None, block_fuse=None, num_blocks=[3, 4, 6, 3], m_channels=32, mul_channel=1,
                 expansion=2, base_width=32, scale=2, embd_dim=192, two_emb_layer=False):
        super().__init__()
        if block is not None or block_fuse is not None or two_emb_layer:
            raise NotImplementedError('ERes2Net: custom blocks / two_emb_layer are not lowered')
        self.input_size, self.embd_dim = input_size, embd_dim
        self.num_blocks, self.m, self.mul, self.expansion = list(num_blocks), m_channels, mul_channel, expansion
        self.base_width, self.scale = base_width, scale
        self.F8 = int(input_size / 8)
        self.stats_dim = self.F8 * m_channels * 8
        if m_channels % 4:
            raise NotImplementedError('m_channels must be a multiple of 4')
        self._check_top()

    def _check_top(self):
        if self.m * 2 * self.mul != self.m * self.expansion:
            raise ValueError('mul_channel * 2 must equal expansion (layer1_downsample in-channels, eres2net.py:211)')

    def _blocks(self):
        inpl = self.m
        for li, nb in enumerate(self.num_blocks, start=1):
            planes = self.m * (2 ** (li - 1))
            width = int(math.floor(planes * (self.base_width / 64.0)))
            for b in range(nb):
                stride = 2 if (li > 1 and b == 0) else 1
                sc = stride != 1 or inpl != planes * self.expansion
                yield f'layer{li}.{b}', li, inpl, planes, width, stride, li >= 3, sc
                inpl = planes * self.expansion

    # ---- reference state-dict layout ----
    def _top_shapes(self, d):
        mc = self.m * self.mul
        d['layer1_downsample.weight'] = (mc * 4, mc * 2, 3, 3)
        d['layer2_downsample.weight'] = (mc * 8, mc * 4, 3, 3)
        d['layer3_downsample.weight'] = (mc * 16, mc * 8, 3, 3)
        _aff_names(d, 'fuse_mode12', mc * 4)
        _aff_names(d, 'fuse_mode123', mc * 8)
        _aff_names(d, 'fuse_mode1234', mc * 16)

    def param_shapes(self):
        d = OrderedDict()
        d['conv1.weight'] = (self.m, 1, 3, 3)
        bn_names(d, 'bn1', self.m)
        for p, li, inpl, planes, w, stride, fuse, sc in self._blocks():
            d[p + '.conv1.weight'] = (w * self.scale, inpl, 1, 1)
            bn_names(d, p + '.bn1', w * self.scale)
            for j in range(self.scale):
                d[f'{p}.convs.{j}.weight'] = (w, w, 3, 3)
            for j in range(self.scale):
                bn_names(d, f'{p}.bns.{j}', w)
            if fuse:
                for j in range(self.scale - 1):
                    _aff_names(d, f'{p}.fuse_models.{j}', w)
            d[p + '.conv3.weight'] = (planes * self.expansion, w * self.scale, 1, 1)
            bn_names(d, p + '.bn3', planes * self.expansion)
            if sc:
                d[p + '.shortcut.0.weight'] = (planes * self.expansion, inpl, 1, 1)
                bn_names(d, p + '.shortcut.1', planes * self.expansion)
        self._top_shapes(d)
        d['seg_1.weight'] = (self.embd_dim, self.stats_dim * self.expansion * 2)
        d['seg_1.bias'] = (self.embd_dim,)
        return d

    # ---- weights ----
    def _pack_aff(self, sd, p, arena, ch):
        """AFF over `ch` channels (zero-padded to chp): cat(x, y) -> inter -> ch."""
        chp = _pad4(ch)
        W0, b0 = fold_conv_bn(sd, p + '.local_att.0.weight', p + '.local_att.1', p + '.local_att.0.bias')   # [inter, 2ch]
        W1, b1 = fold_conv_bn(sd, p + '.local_att.3.weight', p + '.local_att.4', p + '.local_att.3.bias')   # [ch, inter]
        inter = W0.shape[0]
        ip = _pad4(inter)
        W0 = _grp_rows(_grp_cols(W0, ch, chp, 2), inter, ip, 1)
        b0 = _grp_rows(np.asarray(b0, dtype=np.float64).reshape(-1), inter, ip, 1)
        W1 = _grp_rows(_grp_cols(W1, inter, ip, 1), ch, chp, 1)
        b1 = _grp_rows(np.asarray(b1, dtype=np.float64).reshape(-1), ch, chp, 1)
        return dict(w0=arena.add_conv(p + '.w0', W0), b0=arena.add(p + '.b0', b0), w1=arena.add_conv(p + '.w1', W1),
                    b1=arena.add(p + '.b1', b1), inter=ip, ch=chp)

    def _pack_top(self, sd, arena):
        o = self._off
        mc = self.m * self.mul
        for nm in ('layer1_downsample', 'layer2_downsample', 'layer3_downsample'):
            o[nm] = arena.add_conv(nm + '.w', conv2d_weight(sd[nm + '.weight']))
        for nm, ch in (('fuse_mode12', mc * 4), ('fuse_mode123', mc * 8), ('fuse_mode1234', mc * 16)):
            o[nm] = self._pack_aff(sd, nm, arena, ch)

    def _pack(self, sd, arena):
        o, g = self._off, self.scale
        pack_conv_bn(sd, arena, o, 'stem', 'conv1.weight', 'bn1')
        for p, li, inpl, planes, w, stride, fuse, sc in self._blocks():
            wp = _pad4(w)
            W, b = fold_conv_bn(sd, p + '.conv1.weight', p + '.bn1')                       # [g*w, inpl]
            o[p + '.c1'] = dict(w=arena.add_conv(p + '.c1.w', _grp_rows(W, w, wp, g)),
                                b=arena.add(p + '.c1.b', _grp_rows(np.asarray(b).reshape(-1), w, wp, g)))
            for j in range(g):
                W, b = fold_conv_bn(sd, f'{p}.convs.{j}.weight', f'{p}.bns.{j}')            # [w, 9*w], K = (tap, ci)
                W = _grp_rows(_grp_cols(W, w, wp, 9), w, wp, 1)
                o[f'{p}.k{j}'] = dict(w=arena.add_conv(f'{p}.k{j}.w', W),
                                      b=arena.add(f'{p}.k{j}.b', _grp_rows(np.asarray(b).reshape(-1), w, wp, 1)))
            if fuse:
                for j in range(g - 1):
                    o[f'{p}.aff{j}'] = self._pack_aff(sd, f'{p}.fuse_models.{j}', arena, w)
            W, b = fold_conv_bn(sd, p + '.conv3.weight', p + '.bn3')                       # [planes*exp, g*w]
            o[p + '.c3'] = dict(w=arena.add_conv(p + '.c3.w', _grp_cols(W, w, wp, g)), b=arena.add(p + '.c3.b', b))
            if sc:
                pack_conv_bn(sd, arena, o, p + '.sc', p + '.shortcut.0.weight', p + '.shortcut.1')
        self._pack_top(sd, arena)
        C4 = self.m * 8 * self.expansion
        perm = fc_perm(self.F8, C4)
        n = self.F8 * C4
        perm2 = np.concatenate([perm, n + perm])
        o['fc_w'] = arena.add('fc.w', _np64(sd['seg_1.weight'])[:, perm2])
        o['fc_b'] = arena.add('fc.b', sd['seg_1.bias'])

    # ---- program ----
    def _aff(self, pb, e, x, y, rows_per_utt, rows, t, f):
        """xo = x * (1 + tanh(att)) + y * (1 - tanh(att)), att = local_att(cat(x, y)) (eres2net.py:44-50)."""
        a0 = pb.alloc(rows, e['inter'])
        pb.conv(x, a0, e['w0'], x.C + y.C, t, t, Fin=f, Fout=f, bias=e['b0'], act=L.ACT_SILU, src2=y,
                src2_mode=L.SRC2_CONCAT)
        a1 = pb.alloc(rows, e['ch'])
        pb.conv(a0, a1, e['w1'], e['inter'], t, t, Fin=f, Fout=f, bias=e['b1'])
        pb.free(a0)
        out = pb.alloc(rows, e['ch'])
        pb.ew(L.EW_AFF, x, out, rows_per_utt, y=y, att=a1)
        pb.free(a1)
        return out

    def _lower_top(self, pb, layer_out, B):
        """Bottom-up fusion of the four stage outputs (eres2net.py:246-253); returns (map, t, f)."""
        o = self._off
        fused, ft, ff = layer_out[1]
        for li, (ds, aff) in enumerate((('layer1_downsample', 'fuse_mode12'), ('layer2_downsample', 'fuse_mode123'),
                                        ('layer3_downsample', 'fuse_mode1234')), start=2):
            xo, to, fo = layer_out[li]
            assert to == out_len(ft, 3, 2, 1) and fo == out_len(ff, 3, 2, 1)
            rows = B * to * fo
            d = pb.alloc(rows, xo.C)
            pb.conv(fused, d, o[ds], 9 * fused.C, ft, to, Fin=ff, Fout=fo, KT=3, KF=3, sT=2, sF=2, padT=1, padF=1)
            pb.free(fused)
            nf = self._aff(pb, o[aff], xo, d, to * fo, rows, to, fo)
            pb.free(d)
            pb.free(xo)
            fused, ft, ff = nf, to, fo
        return fused, ft, ff

    _KEEP_STAGES = (1, 2, 3)           # stage outputs that the top-level fusion reads again

    def _lower(self, pb, B, T):
        o, g = self._off, self.scale
        x, t, f = lower_stem_c1(pb, o['stem'], B, T, self.input_size, self.m)
        layer_out = {}
        last_li = 1
        for p, li, inpl, planes, w, stride, fuse, sc in self._blocks():
            wp = _pad4(w)
            if li != last_li:
                layer_out[last_li] = (x, t, f)        # stage output; kept alive only if the fusion needs it
                last_li = li
            keep_x = any(x is v[0] for k, v in layer_out.items() if k in self._KEEP_STAGES)
            to, fo = out_len(t, 1, stride, 0), out_len(f, 1, stride, 0)
            rows = B * to * fo
            h = pb.alloc(rows, wp * g)
            pb.conv(x, h, o[p + '.c1']['w'], inpl, t, to, Fin=f, Fout=fo, sT=stride, sF=stride, bias=o[p + '.c1']['b'],
                    act=HT)
            cat = pb.alloc(rows, wp * g)
            for j in range(g):
                e = o[f'{p}.k{j}']
                dst = cat.cols(j * wp, wp)
                kw = dict(Fin=fo, Fout=fo, KT=3, KF=3, padT=1, padF=1, bias=e['b'], act=HT)
                if j == 0:
                    pb.conv(h.cols(0, wp), dst, e['w'], 9 * wp, to, to, **kw)
                elif fuse:
                    fz = self._aff(pb, o[f'{p}.aff{j - 1}'], cat.cols((j - 1) * wp, wp), h.cols(j * wp, wp), to * fo, rows,
                                   to, fo)
                    pb.conv(fz, dst, e['w'], 9 * wp, to, to, **kw)
                    pb.free(fz)
                else:
                    pb.conv(cat.cols((j - 1) * wp, wp), dst, e['w'], 9 * wp, to, to, src2=h.cols(j * wp, wp),
                            src2_mode=L.SRC2_ADD, **kw)
            pb.free(h)
            cout = planes * self.expansion
            if sc:
                res = pb.alloc(rows, cout)
                pb.conv(x, res, o[p + '.sc']['w'], inpl, t, to, Fin=f, Fout=fo, sT=stride, sF=stride,
                        bias=o[p + '.sc']['b'])
            else:
                res = x
            y = pb.alloc(rows, cout)
            pb.conv(cat, y, o[p + '.c3']['w'], wp * g, to, to, Fin=fo, Fout=fo, bias=o[p + '.c3']['b'], res=res,
                    act2=HT)
            pb.free(cat)
            if sc:
                pb.free(res)
            if not keep_x:
                pb.free(x)
            x, t, f = y, to, fo
        layer_out[last_li] = (x, t, f)
        fused, ft, ff = self._lower_top(pb, layer_out, B)
        assert ff == self.F8, 'input_size must be a multiple of 8'
        C4 = fused.C
        flat = View(fused.off, ff * C4, 0, ff * C4)
        stats = pb.alloc(B, 2 * ff * C4)
        pb.colstats(flat, stats, ft, L.STATS_MEAN_STD_TSTP, eps=1e-8)
        pb.free(fused)
        pb.conv(stats, pb.output_view(self.embd_dim, B), o['fc_w'], 2 * ff * C4, 1, 1, bias=o['fc_b'],
                engine=L.ENGINE_FFMA)


class ERes2NetV2(ERes2Net):
    """eres2net.py:383-456: same blocks, base_width 26 by default, only out3 is fused into out4."""

    def __init__(self, input_size, block=None, block_fuse=None, num_blocks=[3, 4, 6, 3], m_channels=32, expansion=2,
                 base_width=26, scale=2, embd_dim=192, two_emb_layer=False):
        super().__init__(input_size, block=block, block_fuse=block_fuse, num_blocks=num_blocks, m_channels=m_channels,
                         mul_channel=1, expansion=expansion, base_width=base_width, scale=scale, embd_dim=embd_dim,
                         two_emb_layer=two_emb_layer)

    def _check_top(self):
        if self.expansion != 2:
            raise ValueError('ERes2NetV2: layer3_ds / fuse34 are built for expansion == 2 (eres2net.py:418-419)')

    def _top_shapes(self, d):
        d['layer3_ds.weight'] = (self.m * 16, self.m * 8, 3, 3)
        _aff_names(d, 'fuse34', self.m * 16)

    def _pack_top(self, sd, arena):
        o = self._off
        o['layer3_ds'] = arena.add_conv('layer3_ds.w', conv2d_weight(sd['layer3_ds.weight']))
        o['fuse34'] = self._pack_aff(sd, 'fuse34', arena, self.m * 16)

    _KEEP_STAGES = (3,)

    def _lower_top(self, pb, layer_out, B):
        o = self._off
        x3, t3, f3 = layer_out[3]
        x4, t4, f4 = layer_out[4]
        rows = B * t4 * f4
        d = pb.alloc(rows, x4.C)
        pb.conv(x3, d, o['layer3_ds'], 9 * x3.C, t3, t4, Fin=f3, Fout=f4, KT=3, KF=3, sT=2, sF=2, padT=1, padF=1)
        pb.free(x3)
        nf = self._aff(pb, o['fuse34'], x4, d, t4 * f4, rows, t4, f4)
        pb.free(d)
        pb.free(x4)
        return nf, t4, f4
