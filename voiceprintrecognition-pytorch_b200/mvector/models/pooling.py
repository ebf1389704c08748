"""Attentive statistics pooling, lowered.  Mirrors mvector/models/pooling.py:68-127 (lengths=None, global_context).

The reference materialises attn = cat([x, mean.repeat(T), std.repeat(T)]) (a [B, 3C, T] copy, 1.4 GB at ECAPA B=256)
and runs a 3C -> A 1x1 conv over it.  Algebraically  W[:, :C] x_t + (W[:, C:2C] mean + W[:, 2C:] std + b)  -- the
second term is a per-utterance bias computed once by a [B, 2C] x [2C, A] product, so the lowered form is:
  stats  = colstats(mean, std)                       [B, 2C]
  ubias  = stats @ W[:, C:3C]^T + b                  [B, A]
  h      = tanh(bn(relu(x @ W[:, :C]^T + ubias)))    [B*T, A]      (TDNNBlock = conv -> ReLU -> BN, then tanh)
  logits = h @ Wc^T + bc                             [B*T, C]
  pooled = softmax_T(logits)-weighted mean / std     [B, 2C]
"""
import numpy as np

from .. import _lib as L
from .base import _np64, bn_affine, bn_names


def asp_shapes(d, p, c, att=128):
    d[p + '.tdnn.conv.conv.weight'] = (att, c * 3, 1)
    d[p + '.tdnn.conv.conv.bias'] = (att,)
    bn_names(d, p + '.tdnn.norm.norm', att)
    d[p + '.conv.conv.weight'] = (c, att, 1)
    d[p + '.conv.conv.bias'] = (c,)


def pack_asp(sd, p, arena, C, perm=None):
    """perm[j] = reference channel held by lowered column j (2-D backbones flatten (f, c) instead of (c, f))."""
    W = _np64(sd[p + '.tdnn.conv.conv.weight'])[:, :, 0]            # [A, 3C]
    A = W.shape[0]
    Wc = _np64(sd[p + '.conv.conv.weight'])[:, :, 0]                # [C, A]
    bc = _np64(sd[p + '.conv.conv.bias'])
    if perm is not None:
        W = np.concatenate([W[:, perm], W[:, C + perm], W[:, 2 * C + perm]], axis=1)
        Wc, bc = Wc[perm], bc[perm]
    s, h = bn_affine(sd, p + '.tdnn.norm.norm')
    return dict(A=A, C=C,
                wx=arena.add_conv(p + '.tdnn.wx', W[:, :C]), wms=arena.add(p + '.tdnn.wms', W[:, C:]),
                b=arena.add(p + '.tdnn.b', sd[p + '.tdnn.conv.conv.bias']),
                s=arena.add(p + '.tdnn.bn_s', s), h=arena.add(p + '.tdnn.bn_h', h),
                wc=arena.add_conv(p + '.conv.w', Wc), bc=arena.add(p + '.conv.b', bc))


def lower_asp(pb, o, x, B, T, pooled):
    """x: View [B*T, C]; pooled: View [B, 2C] (mean ; std)."""
    C, A = o['C'], o['A']
    stats = pb.alloc(B, 2 * C)
    pb.colstats(x, stats, T, L.STATS_MEAN_STD_CLAMP, eps=1e-12)
    ub = pb.alloc(B, A)
    pb.conv(stats, ub, o['wms'], 2 * C, 1, 1, bias=o['b'], engine=L.ENGINE_FFMA)
    h = pb.alloc(B * T, A)
    pb.conv(x, h, o['wx'], C, T, T, ubias=ub, act=L.ACT_RELU, post=(o['s'], o['h']), act2=L.ACT_TANH)
    logits = pb.alloc(B * T, C)
    pb.conv(h, logits, o['wc'], A, T, T, bias=o['bc'])
    pb.asp_pool(x, logits, pooled, T, eps=1e-12)
    for v in (logits, h, ub, stats):
        pb.free(v)


# ---------------------------------------------------------------------------------------------------------------
# The other pooling types of the reference (pooling.py:8-65), selectable through ``pooling_type`` in the yml:
#   TAP  mean over T                         -> one COLSTATS(MEAN)
#   TSP  mean ; unbiased VARIANCE            -> one COLSTATS(MEAN_VAR_UNBIASED)   (pooling.py:44-46 returns var, not std)
#   SAP  softmax_T(W2 tanh(W1 x + b1) + b2)-weighted mean -> two CONVs + ASP_POOL(mean only)
# ---------------------------------------------------------------------------------------------------------------
POOL_TYPES = ('ASP', 'SAP', 'TAP', 'TSP')


def check_pooling_type(pooling_type):
    if pooling_type not in POOL_TYPES:
        raise Exception(f'没有{pooling_type}池化层！')


def pool_width(kind, c):
    return 2 * c if kind in ('ASP', 'TSP') else c


def pool_shapes(d, p, kind, c, att=128):
    if kind == 'ASP':
        asp_shapes(d, p, c, att)
    elif kind == 'SAP':
        d[p + '.linear1.weight'] = (128, c, 1)
        d[p + '.linear1.bias'] = (128,)
        d[p + '.linear2.weight'] = (c, 128, 1)
        d[p + '.linear2.bias'] = (c,)
    return pool_width(kind, c)


def pack_pool(sd, p, kind, arena, C, perm=None):
    if kind == 'ASP':
        return pack_asp(sd, p, arena, C, perm)
    if kind == 'SAP':
        W1 = _np64(sd[p + '.linear1.weight'])[:, :, 0]          # [128, C]
        W2 = _np64(sd[p + '.linear2.weight'])[:, :, 0]          # [C, 128]
        b2 = _np64(sd[p + '.linear2.bias'])
        if perm is not None:
            W1, W2, b2 = W1[:, perm], W2[perm], b2[perm]
        return dict(C=C, A=W1.shape[0], w1=arena.add_conv(p + '.w1', W1), b1=arena.add(p + '.b1', sd[p + '.linear1.bias']),
                    w2=arena.add_conv(p + '.w2', W2), b2=arena.add(p + '.b2', b2))
    return dict(C=C)


def pool_perm(kind, C, perm):
    """Column permutation of the pooled vector when the backbone's channel order is permuted (2-D nets)."""
    if perm is None:
        return None
    return np.concatenate([perm, C + perm]) if kind in ('ASP', 'TSP') else perm


def lower_pool(pb, o, kind, x, B, T, pooled):
    if kind == 'ASP':
        lower_asp(pb, o, x, B, T, pooled)
    elif kind == 'TAP':
        pb.colstats(x, pooled, T, L.STATS_MEAN)
    elif kind == 'TSP':
        if T < 2:
            raise ValueError('TSP pooling needs at least 2 frames (unbiased variance)')
        pb.colstats(x, pooled, T, L.STATS_MEAN_VAR_UNBIASED)
    elif kind == 'SAP':
        C, A = o['C'], o['A']
        h = pb.alloc(B * T, A)
        pb.conv(x, h, o['w1'], C, T, T, bias=o['b1'], act=L.ACT_TANH)
        logits = pb.alloc(B * T, C)
        pb.conv(h, logits, o['w2'], A, T, T, bias=o['b2'])
        pb.asp_pool(x, logits, pooled, T, mean_only=True)
        pb.free(logits)
        pb.free(h)


# ---------------------------------------------------------------------------------------------------------------
# The embedding head shared by ECAPA, TDNN, ResNetSE and Res2Net: pooling -> BN `bn` -> linear `fc` (-> BN `post_bn`).
# The BN(s) and the linear layer are affine, so they collapse into one [embd, width] product folded in fp64 at pack time.
# ---------------------------------------------------------------------------------------------------------------
def head_shapes(d, kind, c, embd, bn, fc, post_bn=None, pool='pooling', att=128, fc_conv1d=False):
    """``fc_conv1d``: the linear layer is a kernel-1 Conv1d (weight [embd, width, 1]) instead of an nn.Linear."""
    width = pool_shapes(d, pool, kind, c, att)
    bn_names(d, bn, width)
    d[fc + '.weight'] = (embd, width, 1) if fc_conv1d else (embd, width)
    d[fc + '.bias'] = (embd,)
    if post_bn is not None:
        bn_names(d, post_bn, embd)


def pack_head(sd, arena, kind, c, bn, fc, post_bn=None, pool='pooling', perm=None):
    """perm: the (f, c) column order of a 2-D backbone's flattened map (conv2d_util.fc_perm), folded into the weights."""
    o = dict(pool=pack_pool(sd, pool, kind, arena, c, perm=perm))
    s, h = bn_affine(sd, bn)
    W = _np64(sd[fc + '.weight'])
    W = W.reshape(W.shape[0], -1)
    b = W @ h + _np64(sd[fc + '.bias'])
    if post_bn is None:             # not an identity post-BN: multiplying by s2 = 1 can still change a -0 into +0
        W = W * s[None, :]
    else:
        s2, h2 = bn_affine(sd, post_bn)
        W, b = s2[:, None] * W * s[None, :], s2 * b + h2
    if perm is not None:
        W = W[:, pool_perm(kind, c, perm)]
    o['w'], o['b'] = arena.add('fc.w', W), arena.add('fc.b', b)
    return o


def lower_head(pb, o, kind, x, B, T, embd):
    """x: View [B*T, C], freed after pooling.  Writes the embeddings [B, embd] and returns the pooled View [B, width]."""
    width = pool_width(kind, x.C)
    pooled = pb.alloc(B, width)
    lower_pool(pb, o['pool'], kind, x, B, T, pooled)
    pb.free(x)
    pb.conv(pooled, pb.output_view(embd, B), o['w'], width, 1, 1, bias=o['b'], engine=L.ENGINE_FFMA)
    return pooled
