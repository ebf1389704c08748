"""Shared helpers for the 2-D (conv2d) backbones.  Activation maps are channel-last [B, T, F, C]: T (time) is the
conv2d W axis and F (frequency) the H axis of the reference's [B, C, F, T] tensors, so that the final
``reshape(B, C*F, T)`` (campplus.py:290-291, resnet_se.py:139) is free: row (b, t) already holds the F*C values,
in (f, c) order instead of the reference's (c, f) -- the permutation is folded into the next layer's weights."""
import numpy as np

from .. import _lib as L
from ..engine import View
from .base import _np64, bn_affine


def conv2d_weight(w):
    """[Cout, Cin, kF, kT] -> [Cout, (kt, kf, ci)]: the K order of the CONV op's gather."""
    w = _np64(w)
    return np.ascontiguousarray(w.transpose(0, 3, 2, 1)).reshape(w.shape[0], -1)


def fold_conv_bn(sd, conv_key, bn_prefix, bias_key=None):
    """conv -> BN (eval) == conv with W * s[n] and bias (b * s + h): returns (W2d fp64, bias fp64)."""
    W = conv2d_weight(sd[conv_key])
    s, h = bn_affine(sd, bn_prefix)
    b = _np64(sd[bias_key]) if bias_key is not None else 0.0
    return W * s[:, None], b * s + h


def pack_conv_bn(sd, arena, o, name, conv_key, bn_prefix):
    """o[name] = the conv ``conv_key`` with its BN folded in, packed as dict(w=..., b=...)."""
    W, b = fold_conv_bn(sd, conv_key, bn_prefix)
    o[name] = dict(w=arena.add_conv(name + '.w', W), b=arena.add(name + '.b', b))


def out_len(n, k, s, pad, dil=1):
    return (n + 2 * pad - dil * (k - 1) - 1) // s + 1


def fc_perm(F8, C):
    """perm[j] for lowered column j = f*C + c  ->  reference flattened channel c*F8 + f."""
    f = np.arange(F8)[:, None]
    c = np.arange(C)[None, :]
    return (c * F8 + f).reshape(-1)


def L_view1(v):
    """The [B*T, F] feature matrix seen as a one-channel [B, T, F, 1] map: row stride 1, one column."""
    return View(v.off, 1, 0, 1)


def lower_stem_c1(pb, e, B, T, F, C, k=3, stride=1, pad=1):
    """The stem on the one-channel feature map: k x k stride-s conv2d (CONV_C1, BN folded in ``e``, ReLU) of the
    [B*T, F] input into a [B, t, f, C] map.  Returns (map, t, f)."""
    x_in = pb.input_view(F, B * T)
    t, f = out_len(T, k, stride, pad), out_len(F, k, stride, pad)
    if t < 1 or f < 1:
        raise ValueError(f'{T} frames x {F} bins is too small for the {k}x{k} stride-{stride} stem')
    x = pb.alloc(B * t * f, C)
    pb.conv(L_view1(x_in), x, e['w'], k * k, T, t, Fin=F, Fout=f, KT=k, KF=k, sT=stride, sF=stride, padT=pad, padF=pad,
            bias=e['b'], act=L.ACT_RELU, c1=True)
    return x, t, f
