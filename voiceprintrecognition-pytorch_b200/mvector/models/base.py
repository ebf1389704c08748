"""Common machinery of the backbone mirrors: state-dict ingestion, BatchNorm folding, program cache."""
from collections import OrderedDict

import numpy as np
import torch

from .. import _lib as L
from ..engine import Engine, PlanBuilder, Program, WeightArena


def _np64(t):
    return t.detach().cpu().double().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, dtype=np.float64)


def bn_affine(sd, prefix, eps=1e-5):
    """Eval-mode BatchNorm as y = x * s + h (fp64): s = gamma / sqrt(running_var + eps), h = beta - mean * s."""
    var = _np64(sd[prefix + '.running_var'])
    mean = _np64(sd[prefix + '.running_mean'])
    gamma = _np64(sd[prefix + '.weight']) if (prefix + '.weight') in sd else np.ones_like(var)
    beta = _np64(sd[prefix + '.bias']) if (prefix + '.bias') in sd else np.zeros_like(var)
    s = gamma / np.sqrt(var + eps)
    return s, beta - mean * s


def bn_names(d, p, c, affine=True):
    if affine:
        d[p + '.weight'] = (c,)
        d[p + '.bias'] = (c,)
    d[p + '.running_mean'] = (c,)
    d[p + '.running_var'] = (c,)
    d[p + '.num_batches_tracked'] = ()


def conv1d_weight(w):
    """[Cout, Cin, k] -> [Cout, k*Cin4] with K index = tap*Cin4 + ci (the gather order of the CONV op).  Cin4 = Cin
    rounded up to a multiple of 4 with zero columns: only a first layer fed by an odd feature dim (Spectrogram's
    n_fft/2+1 bins) is ever padded; its input comes through PlanBuilder.input_view1d."""
    w = _np64(w)
    cin = w.shape[1]
    if cin % 4:
        w = np.concatenate([w, np.zeros((w.shape[0], -cin % 4, w.shape[2]), dtype=w.dtype)], axis=1)
    return np.ascontiguousarray(w.transpose(0, 2, 1)).reshape(w.shape[0], -1)


class Backbone:
    """Base of the model mirrors.  A backbone is *lowered* for a concrete (B, T) into a vp_program; programs are
    cached per shape.  Calling the object runs features [B, T, F] (CUDA fp32) -> embeddings [B, embd_dim]."""

    #: (chunk_k, kc): layers with K > chunk_k accumulate in chunks of kc K elements on the tensor cores (vp_op.tc_kc).  The
    #: tensor core truncates on every accumulate, a bias that adds up coherently through a deep network: the shallow TDNNs
    #: keep single-accumulator GEMMs up to K = 1536, the deep 2-D residual nets override this with shorter chains.
    tc_chunk_policy = (1536, 512)

    #: parameter-name -> shape, filled by subclasses (reference state_dict layout, without the ``0.`` prefix)
    def param_shapes(self):
        raise NotImplementedError

    def _pack(self, sd, arena):
        raise NotImplementedError

    def _lower(self, pb, B, T):
        raise NotImplementedError

    def __init__(self):
        self.engine = None
        self._programs = OrderedDict()
        self._off = {}
        self.engine_pref = L.ENGINE_AUTO
        self.max_cached_programs = 64      # programs are host-side op lists: the workspace is the handle's shared arena
        self.training = False
        self._blob = None
        self._blob_id = None               # identifies this blob on an Engine (Engine.weights_owner)

    # -- nn.Module-ish surface used by the reference's call sites (predict.py:55-63) --
    def eval(self):
        return self

    def to(self, device):
        return self

    def state_dict_keys(self):
        return list(self.param_shapes().keys())

    def load_state_dict(self, state_dict, strict=True, engine=None):
        """Ingest a reference state dict (keys with or without the ``0.`` Sequential prefix).  Returns
        (missing_keys, unexpected_keys) like torch (checkpoint.py:43)."""
        shapes = self.param_shapes()
        sd = {}
        unexpected = []
        for k, v in state_dict.items():
            kk = k[2:] if k.startswith('0.') else k
            if kk in shapes:
                if tuple(v.shape) != tuple(shapes[kk]):
                    raise RuntimeError(f'size mismatch for {k}: {tuple(v.shape)} vs {tuple(shapes[kk])}')
                sd[kk] = v
            else:
                unexpected.append(k)
        missing = [k for k in shapes if k not in sd and not k.endswith('num_batches_tracked')]
        if missing:
            # the reference would silently keep its random init for missing tensors (strict=False); a drop-in that
            # invents weights is worse than failing: refuse.
            raise RuntimeError('missing weights for: ' + ', '.join(missing[:8]) + (' ...' if len(missing) > 8 else ''))
        if engine is not None:
            self.engine = engine
        arena = WeightArena(*self.tc_chunk_policy)
        self._off = {}
        self._pack(sd, arena)
        self._blob = arena.blob()          # uploaded lazily: ingesting weights / lowering needs no GPU
        self._blob_id = object()
        self._arena_index = arena.index
        for p in self._programs.values():
            p.close()
        self._programs.clear()
        return missing, unexpected

    def lower(self, B, T, engine_pref=None):
        """Lower to a PlanBuilder (ops + static memory plan) for a concrete (B, T).  Pure host code."""
        if not self._off:
            raise RuntimeError('load_state_dict() first')
        pb = PlanBuilder(B, self.engine_pref if engine_pref is None else engine_pref)
        self._lower(pb, B, T)
        return pb

    def program(self, B, T):
        if self.engine is None:
            self.engine = Engine()
        if self.engine.weights_owner is not self._blob_id:
            # not uploaded yet, or another model sharing the Engine has uploaded its blob since: the handle refuses
            # every program created before that reload, so drop them and upload ours again
            for p in self._programs.values():
                p.close()
            self._programs.clear()
            self.engine.load_weights(self._blob, owner=self._blob_id)
        key = (B, T, self.engine_pref)
        p = self._programs.get(key)
        if p is None:
            pb = self.lower(B, T)
            p = Program(self.engine, pb)
            self._programs[key] = p
            while len(self._programs) > self.max_cached_programs:
                _, old = self._programs.popitem(last=False)
                old.close()
        else:
            self._programs.move_to_end(key)
        return p

    def __call__(self, feats):
        if not (isinstance(feats, torch.Tensor) and feats.is_cuda):
            raise RuntimeError('backbone input must be a CUDA tensor (no CPU path)')
        feats = feats.contiguous().float()
        B, T, F = feats.shape
        if F != self.input_size:
            raise RuntimeError(f'feature dim {F} != model input_size {self.input_size}')
        emb = torch.empty(B, self.embd_dim, dtype=torch.float32, device=feats.device)
        self.program(B, T).run(feats, emb)
        return emb

    forward = __call__
