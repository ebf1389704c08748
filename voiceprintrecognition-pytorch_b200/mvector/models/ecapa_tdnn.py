"""EcapaTdnn mirror (reference: mvector/models/ecapa_tdnn.py:146-283), lowered to fused sm_90a ops.

Lowering of one SERes2NetBlock (ecapa_tdnn.py:87-143), activations channel-last [B*T, C]:
  t1  = bn(relu(x W1 + b))                                   one CONV (1x1 = dense GEMM)
  y   = Res2Net chain, 7 dependent k3 dilated reflect convs  7 CONVs reading t1 slice (+ previous y slice) in the gather
  t2  = bn(relu(y W2 + b))                                   one CONV
  s   = sigmoid(W_b relu(W_a mean_T(t2)))                    COLSTATS + 2 tiny CONVs (rows = B)
  out = s * t2 + residual  -> written straight into its 512-column slot of the [B*T, 1536] MFA input (no torch.cat)
"""
from collections import OrderedDict

from .. import _lib as L
from .base import Backbone, _np64, bn_affine, bn_names, conv1d_weight
from .pooling import check_pooling_type, head_shapes, lower_head, pack_head


def _tdnn_block_shapes(d, p, cin, cout, k):
    d[p + '.conv.conv.weight'] = (cout, cin, k)
    d[p + '.conv.conv.bias'] = (cout,)
    bn_names(d, p + '.norm.norm', cout)


class EcapaTdnn(Backbone):
    def __init__(self, input_size, embd_dim=192, pooling_type='ASP', activation=None,
                 channels=[512, 512, 512, 512, 1536], kernel_sizes=[5, 3, 3, 3, 1], dilations=[1, 2, 3, 4, 1],
                 attention_channels=128, res2net_scale=8, se_channels=128, global_context=True,
                 groups=[1, 1, 1, 1, 1]):
        super().__init__()
        assert len(channels) == len(kernel_sizes) and len(channels) == len(dilations)
        check_pooling_type(pooling_type)
        self.pooling_type = pooling_type
        self.head_bn = 'asp_bn.norm' if pooling_type == 'ASP' else 'asp_bn'     # ecapa_tdnn.py:224 vs :232,239,246
        if activation is not None or not global_context or any(g != 1 for g in groups):
            raise NotImplementedError('EcapaTdnn: only ReLU / global_context=True / groups=1 are lowered')
        for c in channels[:-1]:
            assert c % res2net_scale == 0
        if channels[-1] != sum(channels[1:-1]):
            raise ValueError('channels[-1] must equal the concatenated SE-Res2 outputs (ecapa_tdnn.py:273-274)')
        self.input_size, self.embd_dim = input_size, embd_dim
        self.channels, self.kernel_sizes, self.dilations = list(channels), list(kernel_sizes), list(dilations)
        self.attention_channels, self.res2net_scale, self.se_channels = attention_channels, res2net_scale, se_channels

    def param_shapes(self):
        d = OrderedDict()
        ch, ks = self.channels, self.kernel_sizes
        _tdnn_block_shapes(d, 'blocks.0', self.input_size, ch[0], ks[0])
        for i in range(1, len(ch) - 1):
            p = f'blocks.{i}'
            cin, c = ch[i - 1], ch[i]
            _tdnn_block_shapes(d, p + '.tdnn1', cin, c, 1)
            w = c // self.res2net_scale
            for j in range(self.res2net_scale - 1):
                _tdnn_block_shapes(d, f'{p}.res2net_block.blocks.{j}', w, w, ks[i])
            _tdnn_block_shapes(d, p + '.tdnn2', c, c, 1)
            d[p + '.se_block.conv1.conv.weight'] = (self.se_channels, c, 1)
            d[p + '.se_block.conv1.conv.bias'] = (self.se_channels,)
            d[p + '.se_block.conv2.conv.weight'] = (c, self.se_channels, 1)
            d[p + '.se_block.conv2.conv.bias'] = (c,)
            if cin != c:
                d[p + '.shortcut.conv.weight'] = (c, cin, 1)
                d[p + '.shortcut.conv.bias'] = (c,)
        _tdnn_block_shapes(d, 'mfa', ch[-1], ch[-1], ks[-1])
        head_shapes(d, self.pooling_type, ch[-1], self.embd_dim, self.head_bn, 'fc.conv', pool='asp',
                    att=self.attention_channels, fc_conv1d=True)
        return d

    # ---- weights ----
    def _pack_tdnn_block(self, sd, p, arena):
        s, h = bn_affine(sd, p + '.norm.norm')
        return dict(w=arena.add_conv(p + '.w', conv1d_weight(sd[p + '.conv.conv.weight'])),
                    b=arena.add(p + '.b', sd[p + '.conv.conv.bias']),
                    s=arena.add(p + '.bn_s', s), h=arena.add(p + '.bn_h', h))

    def _pack(self, sd, arena):
        o = self._off
        ch = self.channels
        o['stem'] = self._pack_tdnn_block(sd, 'blocks.0', arena)
        for i in range(1, len(ch) - 1):
            p = f'blocks.{i}'
            blk = dict(tdnn1=self._pack_tdnn_block(sd, p + '.tdnn1', arena),
                       tdnn2=self._pack_tdnn_block(sd, p + '.tdnn2', arena),
                       res2=[self._pack_tdnn_block(sd, f'{p}.res2net_block.blocks.{j}', arena)
                             for j in range(self.res2net_scale - 1)],
                       se_w1=arena.add(p + '.se.w1', _np64(sd[p + '.se_block.conv1.conv.weight'])[:, :, 0]),
                       se_b1=arena.add(p + '.se.b1', sd[p + '.se_block.conv1.conv.bias']),
                       se_w2=arena.add(p + '.se.w2', _np64(sd[p + '.se_block.conv2.conv.weight'])[:, :, 0]),
                       se_b2=arena.add(p + '.se.b2', sd[p + '.se_block.conv2.conv.bias']))
            if (p + '.shortcut.conv.weight') in sd:
                blk['sc_w'] = arena.add_conv(p + '.sc.w', _np64(sd[p + '.shortcut.conv.weight'])[:, :, 0])
                blk['sc_b'] = arena.add(p + '.sc.b', sd[p + '.shortcut.conv.bias'])
            o[p] = blk
        o['mfa'] = self._pack_tdnn_block(sd, 'mfa', arena)
        o['head'] = pack_head(sd, arena, self.pooling_type, ch[-1], self.head_bn, 'fc.conv', pool='asp')

    # ---- program ----
    def _tdnn_block(self, pb, src, dst, w, T, k=1, dil=1, src2=None):
        pad = dil * (k - 1) // 2
        pb.conv(src, dst, w['w'], k * src.C, T, T, KT=k, dT=dil, padT=pad, pad_mode=L.PAD_REFLECT, bias=w['b'],
                act=L.ACT_RELU, post=(w['s'], w['h']), src2=src2, src2_mode=L.SRC2_ADD if src2 is not None else L.SRC2_NONE)

    def _lower(self, pb, B, T):
        ch, ks, dl = self.channels, self.kernel_sizes, self.dilations
        M = B * T
        o = self._off
        for i, k in enumerate(ks):
            if dl[i] * (k - 1) // 2 >= T:
                raise ValueError(f'{T} frames is too short for reflect padding {dl[i] * (k - 1) // 2}')
        x_in = pb.input_view1d(self.input_size, M, T)
        x0 = pb.alloc(M, ch[0])
        self._tdnn_block(pb, x_in, x0, o['stem'], T, ks[0], dl[0])
        if x_in.off != L.BUF_INPUT:
            pb.free(x_in)
        cat = pb.alloc(M, ch[-1])
        xin, coff = x0, 0
        sc = self.res2net_scale
        for i in range(1, len(ch) - 1):
            blk = o[f'blocks.{i}']
            c = ch[i]
            w = c // sc
            t1 = pb.alloc(M, c)
            self._tdnn_block(pb, xin, t1, blk['tdnn1'], T)
            y = pb.alloc(M, c)
            pb.ew(L.EW_COPY, t1.cols(0, w), y.cols(0, w), T)
            # Res2Net chain (ecapa_tdnn.py Res2NetBlock.forward): y_j = block_j(x_j + y_{j-1}).  The add rides in conv
            # j's gather as a second source (two loads per element), not in conv j-1's epilogue as an in-place add
            # (vp_op.sum): that read-modify-write lengthens the epilogue, which at a few tiles per CTA is exposed at every
            # tile hand-over.
            for j in range(1, sc):
                self._tdnn_block(pb, t1.cols(j * w, w), y.cols(j * w, w), blk['res2'][j - 1], T, ks[i], dl[i],
                                 src2=y.cols((j - 1) * w, w) if j >= 2 else None)
            pb.free(t1)
            t2 = pb.alloc(M, c)
            self._tdnn_block(pb, y, t2, blk['tdnn2'], T)
            pb.free(y)
            sq = pb.alloc(B, c)
            pb.colstats(t2, sq, T, L.STATS_MEAN)
            g1 = pb.alloc(B, self.se_channels)
            pb.conv(sq, g1, blk['se_w1'], c, 1, 1, bias=blk['se_b1'], act=L.ACT_RELU, engine=L.ENGINE_FFMA)
            g2 = pb.alloc(B, c)
            pb.conv(g1, g2, blk['se_w2'], self.se_channels, 1, 1, bias=blk['se_b2'], act=L.ACT_SIGMOID,
                    engine=L.ENGINE_FFMA)
            res = xin
            if 'sc_w' in blk:
                res = pb.alloc(M, c)
                pb.conv(xin, res, blk['sc_w'], xin.C, T, T, bias=blk['sc_b'])
            out = cat.cols(coff, c)
            pb.ew(L.EW_GATE_RES, t2, out, T, gate=g2, res=res)
            if 'sc_w' in blk:
                pb.free(res)
            for v in (g2, g1, sq, t2):
                pb.free(v)
            if i == 1:
                pb.free(x0)
            pb.tap(f'block{i}', out, M)
            xin, coff = out, coff + c
        xm = pb.alloc(M, ch[-1])
        self._tdnn_block(pb, cat, xm, o['mfa'], T, ks[-1], dl[-1])
        pb.free(cat)
        pb.tap('mfa', xm, M)
        pb.tap('pooled', lower_head(pb, o['head'], self.pooling_type, xm, B, T, self.embd_dim), B)
