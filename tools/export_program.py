"""Export a lowered program for a C / C++ host (examples/embed_from_c.c): the packed weight arena plus the vp_op list of
one (model, B, T), in one little-endian file.  Needs no GPU (lowering and packing are host work).

    python tools/export_program.py --model EcapaTdnn --feature-dim 80 --batch 8 --frames 298 --out /tmp/ecapa_b8.vpb \
        [--model-args '{"embd_dim": 192}'] [--state-dict model.pth | --seed 0]

File layout: char magic[8] = "VPB200P1"; int32 abi, sizeof_op, n_ops, B, T, F, embd_dim, reserved; uint64 workspace_bytes,
input_floats, output_floats, weights_bytes; vp_op ops[n_ops]; float weights[weights_bytes / 4]."""
import argparse
import ctypes as C
import json
import struct
import sys

import numpy as np

sys.path.insert(0, '.')
MAGIC = b'VPB200P1'


def export(model, B, T, path):
    from mvector import _lib as L
    pb = model.lower(B, T)
    blob = np.ascontiguousarray(model._blob, dtype=np.float32)
    pb.finalize()
    ops = (L.Op * len(pb.ops))(*pb.ops)
    with open(path, 'wb') as f:
        f.write(MAGIC)
        f.write(struct.pack('<8i', L.ABI_VERSION, C.sizeof(L.Op), len(pb.ops), B, T, model.input_size, model.embd_dim, 0))
        f.write(struct.pack('<4Q', max(pb.peak, 256), pb.in_floats, pb.out_floats, blob.nbytes))
        f.write(bytes(ops))
        f.write(blob.tobytes())
    return pb, blob


def load(path):
    """-> dict(header fields, ops = list of _lib.Op, weights = float32 array): the inverse of export (tests)."""
    from mvector import _lib as L
    raw = open(path, 'rb').read()
    assert raw[:8] == MAGIC
    abi, szop, n_ops, B, T, F, embd, _ = struct.unpack_from('<8i', raw, 8)
    ws, inf, outf, wbytes = struct.unpack_from('<4Q', raw, 40)
    assert szop == C.sizeof(L.Op)
    off = 72
    ops = [L.Op.from_buffer_copy(raw, off + i * szop) for i in range(n_ops)]
    off += n_ops * szop
    weights = np.frombuffer(raw, dtype=np.float32, count=wbytes // 4, offset=off)
    assert off + wbytes == len(raw)
    return dict(abi=abi, B=B, T=T, F=F, embd_dim=embd, workspace_bytes=ws, input_floats=inf, output_floats=outf, ops=ops,
                weights=weights)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--model', default='EcapaTdnn')
    ap.add_argument('--model-args', default='{}')
    ap.add_argument('--feature-dim', type=int, default=80)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--frames', type=int, default=298)
    ap.add_argument('--state-dict', default=None, help="reference model.pth ('0.*' keys); default: seeded random weights")
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', required=True)
    a = ap.parse_args()
    import torch
    from mvector.models import build_model
    from mvector.utils.utils import dict_to_object
    margs = json.loads(a.model_args)
    model = build_model(a.feature_dim, dict_to_object({'model_conf': {'model': a.model, 'model_args': margs}}))
    if a.state_dict:
        model.load_state_dict(torch.load(a.state_dict, map_location='cpu', weights_only=False))
    else:
        from oracle import models as om                 # dev tool only: seeded weights for demos
        model.load_state_dict({'0.' + k: v for k, v in om.random_state_dict(a.model, a.feature_dim, seed=a.seed, **margs).items()})
    pb, blob = export(model, a.batch, a.frames, a.out)
    print(f'{a.out}: {len(pb.ops)} ops, workspace {pb.peak / 2**20:.1f} MiB, weights {blob.nbytes / 2**20:.1f} MiB')


if __name__ == '__main__':
    main()
