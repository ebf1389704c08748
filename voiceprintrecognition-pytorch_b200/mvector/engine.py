"""Host-side runtime over the C ABI: device handle, packed weight arena, static memory planner and the program
builder the model mirrors (mvector/models/*.py) lower themselves with.

torch is used for device memory, streams and (multi-GPU) torch.distributed only; every kernel on the path is in
libvpb200.so.
"""
import ctypes as C
import os
from collections import OrderedDict

import numpy as np
import torch

from . import _lib as L

ALIGN = 256  # bytes; every workspace buffer / weight tensor starts on a 256 B boundary
TC_F16 = os.environ.get('VPB_TC_F16', '1') != '0'   # pack the fp16 two-term weight images (VP_ENGINE_TC16); VPB_TC_F16=0: tf32 only


def _check(handle, rc):
    if rc != L.VP_OK:
        msg = L.lib().vp_last_error(handle).decode('utf-8', 'replace') if handle else ''
        raise L.VpError(rc, msg)


class Engine:
    """One per (process, device): owns the vp_handle, the weight arena and the front-end state."""

    def __init__(self, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError('CUDA device required: the vpb200 path has no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device() if device is None else device)
        self._h = C.c_void_p()
        rc = L.lib().vp_create(self.device.index, C.byref(self._h))
        if rc != L.VP_OK:
            raise L.VpError(rc, 'vp_create failed (needs an sm_90 GPU: H100)')
        self._programs = []
        self.weights_owner = None       # which caller's blob the handle holds (load_weights(owner=...))

    @property
    def handle(self):
        return self._h

    def stream_ptr(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def load_weights(self, blob, owner=None):
        """Upload a weight blob, replacing the previous one: every Program created before it is refused from then on
        (vp_weights_load).  ``owner`` records whose blob the handle now holds, so models sharing one Engine can tell
        whether theirs is still resident (Backbone.program)."""
        blob = np.ascontiguousarray(blob, dtype=np.float32)
        self.weights_owner = None
        _check(self._h, L.lib().vp_weights_load(self._h, blob.ctypes.data_as(C.c_void_p), blob.nbytes))
        self.weights_owner = owner

    def cosine_scores(self, a, b):
        """[n, D] x [m, D] -> device tensor [n, m] of cosine similarities (vp_cosine_scores); inputs: numpy / torch."""
        ta = torch.as_tensor(a, dtype=torch.float32).to(self.device).contiguous()
        tb = torch.as_tensor(b, dtype=torch.float32).to(self.device).contiguous()
        if ta.dim() == 1:
            ta = ta.unsqueeze(0)
        if tb.dim() == 1:
            tb = tb.unsqueeze(0)
        assert ta.shape[1] == tb.shape[1]
        out = torch.empty(ta.shape[0], tb.shape[0], dtype=torch.float32, device=self.device)
        _check(self._h, L.lib().vp_cosine_scores(self._h, C.c_void_p(ta.data_ptr()), ta.shape[0], C.c_void_p(tb.data_ptr()),
                                                 tb.shape[0], ta.shape[1], C.c_void_p(out.data_ptr()), self.stream_ptr()))
        return out

    # ---- spectral stage of the diarization clustering (csrc/spectral.cu) ----
    def spectral_scratch(self, n):
        """Device scratch for spectral_laplacian / sym_tridiag at size n (uint8 tensor)."""
        return torch.empty(int(L.lib().vp_spectral_scratch_bytes(self._h, n)), dtype=torch.uint8, device=self.device)

    def spectral_laplacian(self, X, n_drop, scratch=None):
        """[n, D] embeddings -> device float64 [n, n] unnormalised Laplacian of the pruned cosine affinity
        (vp_spectral_laplacian)."""
        tx = torch.as_tensor(X, dtype=torch.float32).to(self.device).contiguous()
        n, D = tx.shape
        scratch = self.spectral_scratch(n) if scratch is None else scratch
        Lm = torch.empty(n, n, dtype=torch.float64, device=self.device)
        _check(self._h, L.lib().vp_spectral_laplacian(self._h, C.c_void_p(tx.data_ptr()), n, D, int(n_drop),
                                                      C.c_void_p(Lm.data_ptr()), C.c_void_p(scratch.data_ptr()),
                                                      self.stream_ptr()))
        return Lm

    def sym_tridiag(self, A, scratch=None):
        """In place on the device float64 symmetric A [n, n]: Householder reduction to tridiag(d, e); -> device
        (d [n], e [n-1], tau [n-1]), the reflectors stay in A (vp_sym_tridiag)."""
        assert A.dtype == torch.float64 and A.is_contiguous() and A.shape[0] == A.shape[1]
        n = A.shape[0]
        scratch = self.spectral_scratch(n) if scratch is None else scratch
        d = torch.empty(n, dtype=torch.float64, device=self.device)
        e = torch.empty(max(n - 1, 1), dtype=torch.float64, device=self.device)
        tau = torch.empty(max(n - 1, 1), dtype=torch.float64, device=self.device)
        _check(self._h, L.lib().vp_sym_tridiag(self._h, C.c_void_p(A.data_ptr()), n, C.c_void_p(d.data_ptr()),
                                               C.c_void_p(e.data_ptr()), C.c_void_p(tau.data_ptr()),
                                               C.c_void_p(scratch.data_ptr()), self.stream_ptr()))
        return d, e[:n - 1], tau[:n - 1]

    def sym_tridiag_apply_q(self, A, tau, Z):
        """Z [n, k] (numpy / torch) -> device float64 Q Z with the reflectors sym_tridiag left in A, tau."""
        tz = torch.as_tensor(Z, dtype=torch.float64).to(self.device).contiguous().clone()
        n, k = tz.shape
        tau_p = tau.data_ptr() if tau.numel() else A.data_ptr()
        _check(self._h, L.lib().vp_sym_tridiag_apply_q(self._h, C.c_void_p(A.data_ptr()), C.c_void_p(tau_p), n,
                                                       C.c_void_p(tz.data_ptr()), k, self.stream_ptr()))
        return tz

    def spectral_embedding(self, X, n_drop, n_eig, k_fn):
        """SpectralCluster's spectral stage: embeddings X [n, D] -> (the n_eig smallest eigenvalues of the pruned-affinity
        Laplacian, the eigenvectors of the first k = k_fn(eigenvalues) of them [n, k]), numpy float64.

        Laplacian, Householder reduction and back-transformation run on the device in fp64; the tridiagonal
        eigenproblem between them -- 2n numbers down, [n, k] up, O(n k) work -- is solved here by LAPACK's bisection and
        inverse iteration (stebz / stein), which resolve clustered eigenvalues such as those of disconnected graph
        components.  That split is by design, like k-means staying on the host; there is no CPU fallback for the O(n^3)
        part."""
        import scipy.linalg
        n = len(X)
        scratch = self.spectral_scratch(n)
        A = self.spectral_laplacian(X, n_drop, scratch)
        d, e, tau = self.sym_tridiag(A, scratch)
        d, e = d.cpu().numpy(), e.cpu().numpy()
        if n == 1:
            lam = d.copy()
            k = k_fn(lam)
            return lam, np.ones((1, k))
        lam = scipy.linalg.eigh_tridiagonal(d, e, eigvals_only=True, select='i', select_range=(0, n_eig - 1))
        k = k_fn(lam)
        _, Zt = scipy.linalg.eigh_tridiagonal(d, e, select='i', select_range=(0, k - 1))
        return lam, self.sym_tridiag_apply_q(A, tau, Zt).cpu().numpy()

    # ---- input conditioning (csrc/condition.cu) ----
    def _tap_offsets(self, pairs):
        """Offsets (float64 elements) of the per-phase tap tables of ``pairs`` in the engine's device tap table; a pair
        seen for the first time is designed on the host (audio.polyphase_taps) and the table uploaded again."""
        from .audio import polyphase_taps
        if not hasattr(self, '_taps'):
            self._taps, self._tap_off, self._taps_dev = [], {}, None
        new = [p for p in pairs if p not in self._tap_off]
        for p in new:
            self._tap_off[p] = sum(t.size for t in self._taps)
            self._taps.append(polyphase_taps(*p)[0])
        if new or self._taps_dev is None:
            self._taps_dev = torch.from_numpy(np.concatenate(self._taps) if self._taps else np.zeros(1)).to(self.device)
        return self._tap_off

    def condition_plan(self, n_in, rates, target_rate, target_db=None, max_gain_db=300.0):
        """Host plan of one conditioning call over rows with ``n_in`` native samples at ``rates`` (ConditionPlan)."""
        return ConditionPlan(self, n_in, rates, target_rate, target_db, max_gain_db)

    def condition(self, wave, n_in, rates, target_rate, target_db=None, max_gain_db=300.0):
        """_load_audio's resample + dB normalisation of a device batch: ``wave`` CUDA float32 [B, in_ld], row b holding
        ``n_in[b]`` samples at ``rates[b]`` Hz.  Rows are resampled to ``target_rate`` where the rate differs
        (vp_resample, bit-identical to AudioSegment.resample), then normalised to ``target_db`` when it is given
        (vp_gain_normalize).  -> (y [B, max n_out] zero padded, n_out int64 numpy [B], flags device int32 [B] or None:
        1 where the gain exceeds ``max_gain_db``; ``ConditionPlan.check`` raises AudioSegment.normalize's ValueError)."""
        assert wave.is_cuda and wave.dtype == torch.float32 and wave.dim() == 2 and wave.is_contiguous()
        plan = self.condition_plan(n_in, rates, target_rate, target_db, max_gain_db)
        B = wave.shape[0]
        if plan.resample:
            y = torch.empty(B, max(int(plan.n_out.max()), 1), dtype=torch.float32, device=self.device)
        else:
            y = wave.clone()
        flags = torch.empty(B, dtype=torch.int32, device=self.device) if plan.gain else None
        plan.run(wave, wave.shape[1], y, y.shape[1], 0, B, flags, plan.scratch(B, y.shape[1]))
        return y, plan.n_out, flags

    # ---- diarization front (csrc/segment.cu) ----
    def frame_energy(self, wave, n, hop):
        """VAD frame energies of the first ``n`` samples of the CUDA float32 row ``wave`` -> device float64 [n // hop],
        bit-identical to AudioSegment.frame_energy (vp_frame_energy)."""
        assert wave.is_cuda and wave.dtype == torch.float32 and wave.is_contiguous() and 0 <= n <= wave.numel()
        out = torch.empty(n // hop, dtype=torch.float64, device=self.device)
        _check(self._h, L.lib().vp_frame_energy(self._h, C.c_void_p(wave.data_ptr()), int(n), int(hop),
                                                C.c_void_p(out.data_ptr()), self.stream_ptr()))
        return out

    def gather_windows(self, src, offset, valid, ld, dst, stream=None):
        """Row i of ``dst`` [len(offset), ld] (CUDA float32, contiguous) <- ``src[offset[i]:offset[i] + valid[i]]``, zero
        filled to ``ld`` samples (vp_gather_windows); ``offset`` / ``valid`` CUDA int64 / int32 vectors."""
        n = offset.numel()
        assert offset.dtype == torch.int64 and valid.dtype == torch.int32 and valid.numel() == n
        assert src.is_cuda and src.dtype == torch.float32 and dst.dtype == torch.float32 and dst.numel() >= n * ld
        sp = self.stream_ptr() if stream is None else C.c_void_p(stream.cuda_stream)
        _check(self._h, L.lib().vp_gather_windows(self._h, C.c_void_p(src.data_ptr()), C.c_void_p(offset.data_ptr()),
                                                  C.c_void_p(valid.data_ptr()), n, int(ld), C.c_void_p(dst.data_ptr()), sp))

    # ---- FLAC decoding (csrc/flac.cu) ----
    def decode_flac(self, streams, infos=None, names=None, ld=None, check=True):
        """Native FLAC streams (bytes-like each; ``infos`` their flac.StreamInfo, parsed here when omitted) -> (rows CUDA
        float32 [B, ld] at the native rates, zero filled past each stream's length, status CUDA int32 [B]): one
        vp_flac_decode, every row mixed to mono exactly as audio.pcm_to_mono mixes the same integers.  ``ld`` defaults to
        the longest stream.  With ``check`` a non-zero status raises ValueError naming the item (``names``, default
        'item i'); that waits for the decode."""
        from .flac import FlacBatch, parse_streaminfo
        infos = [parse_streaminfo(s) for s in streams] if infos is None else infos
        return self.decode_batch(FlacBatch(streams, infos, self.device, names), ld, check)

    def decode_flac_into(self, batch, out, ld, status, stream=None):
        """vp_flac_decode of a flac.FlacBatch into ``out``, contiguous CUDA float32 holding B rows of ``ld`` (a matrix or a
        flat staging slot), and the int32 ``status`` on ``stream`` (default: the current stream)."""
        B = len(batch)
        if B == 0:
            return
        assert out.dtype == torch.float32 and out.is_cuda and out.is_contiguous() and out.numel() >= B * ld
        assert status.dtype == torch.int32 and status.is_cuda and status.numel() >= B
        stream = torch.cuda.current_stream(self.device) if stream is None else stream
        with torch.cuda.stream(stream):              # the scratch belongs to the stream the decode runs on
            scratch = torch.empty(max(int(L.lib().vp_flac_scratch_bytes(self._h, B, batch.nbytes, batch.max_frames)), 1),
                                  dtype=torch.uint8, device=self.device)
        sp = C.c_void_p(stream.cuda_stream)
        _check(self._h, L.lib().vp_flac_decode(
            self._h, C.c_void_p(batch.data.data_ptr()), C.c_void_p(batch.stream_off_dev.data_ptr()),
            C.c_void_p(batch.frame_off_dev.data_ptr()), C.c_void_p(batch.info.data_ptr()), B,
            C.c_void_p(out.data_ptr()), int(ld), C.c_void_p(status.data_ptr()), C.c_void_p(scratch.data_ptr()),
            batch.nbytes, batch.max_frames, sp))

    # ---- PCM container conversion (csrc/pcm.cu) ----
    def decode_pcm(self, files, infos=None, names=None, ld=None, check=True):
        """Uncompressed PCM container files (bytes-like each; ``infos`` their pcm.PcmInfo, parsed here when omitted) ->
        (rows CUDA float32 [B, ld] at the native rates, zero filled past each file's length, status CUDA int32 [B]): one
        vp_pcm_decode, every row bit-identical to pcm.to_mono.  ``ld`` defaults to the longest file.  With ``check`` a
        non-zero status raises ValueError naming the item (``names``, default 'item i'); that waits for the
        conversion."""
        from .pcm import PcmBatch, parse_header
        infos = [parse_header(f) for f in files] if infos is None else infos
        return self.decode_batch(PcmBatch(files, infos, self.device, names), ld, check)

    def decode_pcm_into(self, batch, out, ld, status, stream=None):
        """vp_pcm_decode of a pcm.PcmBatch into ``out``, contiguous CUDA float32 holding B rows of ``ld`` (a matrix or a
        flat staging slot), and the int32 ``status`` on ``stream`` (default: the current stream)."""
        B = len(batch)
        if B == 0:
            return
        assert out.dtype == torch.float32 and out.is_cuda and out.is_contiguous() and out.numel() >= B * ld
        assert status.dtype == torch.int32 and status.is_cuda and status.numel() >= B
        stream = torch.cuda.current_stream(self.device) if stream is None else stream
        _check(self._h, L.lib().vp_pcm_decode(
            self._h, C.c_void_p(batch.data.data_ptr()), batch.nbytes, C.c_void_p(batch.info.data_ptr()), B,
            C.c_void_p(out.data_ptr()), int(ld), C.c_void_p(status.data_ptr()), C.c_void_p(stream.cuda_stream)))

    def decode_batch(self, batch, ld=None, check=True):
        """An audio.EncodedBatch (flac.FlacBatch, pcm.PcmBatch) decoded by its codec's kernel -> (rows CUDA float32
        [B, ld] at the native rates, zero filled past each item's length, status CUDA int32 [B]); ``ld`` defaults to the
        longest item.  With ``check`` a non-zero status raises ValueError naming the item; that waits for the decode."""
        from .audio import check_status
        B = len(batch)
        ld = int(batch.lengths.max()) if ld is None and B else int(ld or 0)
        out = torch.empty(B, ld, dtype=torch.float32, device=self.device)
        status = torch.empty(B, dtype=torch.int32, device=self.device)
        batch.decode_into(self, out, ld, status)
        if check:
            check_status(status.cpu().numpy(), batch.names, batch.label, batch.unit)
        return out, status

    # ---- verification metrics (csrc/verify.cu) ----
    def verify(self, scores, labels=None, trial_labels=None, enroll_labels=None, p_target=0.01, c_miss=1, c_fa=1,
               sorted_out=False):
        """vp_verify_metrics on a flat score list: -> (vp_verify_result, sorted scores, sorted label codes), the last
        two device tensors with ``sorted_out`` else None.  Labels: ``labels`` [n] (flat form) or ``trial_labels`` /
        ``enroll_labels`` with n = n_trials * n_enroll, score i = trial i // n_enroll against enrolment i % n_enroll."""
        ts = torch.as_tensor(scores, dtype=torch.float32).to(self.device).contiguous().reshape(-1)
        n = ts.numel()

        def dev_i32(x):
            return None if x is None else torch.as_tensor(np.asarray(x), dtype=torch.int32).to(self.device).contiguous().reshape(-1)

        tl, tt, te = dev_i32(labels), dev_i32(trial_labels), dev_i32(enroll_labels)
        if tl is not None and tl.numel() != n:
            raise ValueError(f'{n} scores but {tl.numel()} labels')
        def ptr(t):                    # NULL for an absent tensor; an empty label vector still selects its form
            return C.c_void_p(None if t is None else (t.data_ptr() or 1))

        scratch = torch.empty(max(int(L.lib().vp_verify_scratch_bytes(self._h, n)), 1), dtype=torch.uint8,
                              device=self.device)
        res_dev = torch.empty(C.sizeof(L.VerifyResult), dtype=torch.uint8, device=self.device)
        ss = torch.empty(n, dtype=torch.float32, device=self.device) if sorted_out else None
        sl = torch.empty(n, dtype=torch.uint8, device=self.device) if sorted_out else None
        _check(self._h, L.lib().vp_verify_metrics(
            self._h, ptr(ts), n, ptr(tl), ptr(tt), 0 if tt is None else tt.numel(), ptr(te),
            0 if te is None else te.numel(), float(p_target), float(c_miss), float(c_fa), C.c_void_p(scratch.data_ptr()),
            ptr(ss), ptr(sl), C.c_void_p(res_dev.data_ptr()), self.stream_ptr()))
        res = L.VerifyResult.from_buffer_copy(res_dev.cpu().numpy().tobytes())      # the one synchronise
        return res, ss, sl

    def verification_metrics(self, scores_dev, labels=None, trial_labels=None, enroll_labels=None, p_target=0.01,
                             c_miss=1, c_fa=1, curves=False):
        """EER / minDCF / threshold of a score list on the device (compute_fnr_fpr + compute_eer + compute_dcf,
        metric/metrics.py) -> (eer, min_dcf, threshold), plus (fnr, fpr, thresholds) numpy arrays with ``curves``.
        Raises IndexError where compute_eer does."""
        from .metric.verification import curves_from_sorted, metrics_from_result
        res, ss, sl = self.verify(scores_dev, labels, trial_labels, enroll_labels, p_target, c_miss, c_fa, curves)
        out = metrics_from_result(res, p_target, c_miss, c_fa)
        if not curves:
            return out
        return out + curves_from_sorted(ss.cpu().numpy(), sl.cpu().numpy())

    def close(self):
        if self._h:
            for p in list(self._programs):
                p.close()
            L.lib().vp_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ConditionPlan:
    """Host plan of one conditioning call: per-row (up, down), output lengths and tap offsets, uploaded to the device
    ONCE (one small copy before any kernel of the call is enqueued); ``run`` then conditions any row range [lo, hi) with
    pointer offsets into it, so a staging loop enqueues no further copy."""

    def __init__(self, engine, n_in, rates, target_rate, target_db=None, max_gain_db=300.0):
        from .audio import resample_ratio, resampled_length
        self.engine = engine
        self.target_rate = int(target_rate)
        self.target_db, self.max_gain_db = target_db, float(max_gain_db)
        self.n_in = np.asarray(n_in, dtype=np.int64).reshape(-1)
        B = self.n_in.size
        self.rates = np.broadcast_to(np.asarray(rates, dtype=np.int64), (B,))
        ratio = {r: resample_ratio(r, target_rate) for r in set(self.rates.tolist())}
        self.up = np.fromiter((ratio[r][0] for r in self.rates.tolist()), dtype=np.int32, count=B)
        self.down = np.fromiter((ratio[r][1] for r in self.rates.tolist()), dtype=np.int32, count=B)
        self.n_out = resampled_length(self.n_in, self.up, self.down)
        self.rs_rows = self.up != self.down
        self.resample = bool(self.rs_rows.any())
        self.gain = target_db is not None
        self._meta = None
        if not (self.resample or self.gain):
            return
        tap_off = np.zeros(B, dtype=np.int64)
        if self.resample:
            offs = engine._tap_offsets(sorted({p for p, rs in zip(zip(self.up.tolist(), self.down.tolist()), self.rs_rows)
                                               if rs}))
            tap_off = np.fromiter((offs.get(p, 0) for p in zip(self.up.tolist(), self.down.tolist())), dtype=np.int64,
                                  count=B)
        # one buffer: n_in, n_out, tap_off (int64 [B] each), up, down (int32 [B] each)
        buf = np.concatenate([self.n_in.view(np.uint8), self.n_out.view(np.uint8), tap_off.view(np.uint8),
                              self.up.view(np.uint8), self.down.view(np.uint8)])
        self._meta = torch.from_numpy(buf).to(engine.device)
        self._base = self._meta.data_ptr()
        self._B = B

    def rows_resampled(self, lo, hi):
        return bool(self.rs_rows[lo:hi].any())

    def scratch(self, rows, ld):
        """Device scratch of the gain for ``rows`` rows of leading dimension ``ld`` (None without gain)."""
        if not self.gain:
            return None
        nb = int(L.lib().vp_gain_scratch_bytes(self.engine.handle, rows, ld))
        return torch.empty(max(nb, 1), dtype=torch.uint8, device=self.engine.device)

    def _ptr(self, block, itemsize, lo):
        return C.c_void_p(self._base + 8 * self._B * min(block, 3) + 4 * self._B * max(block - 3, 0) + itemsize * lo)

    def run(self, x, in_ld, y, out_ld, lo, hi, flags, scratch, stream=None):
        """Condition rows lo..hi: ``x`` native rows [hi - lo, in_ld] -> ``y`` [hi - lo, out_ld] (device float32; with
        nothing to resample in the range ``y`` must already hold the rows, x is not read), then the gain in place on
        ``y`` with the rows' flags written to ``flags[lo:hi]`` (a device int32 tensor over ALL rows of the plan)."""
        eng = self.engine
        sp = eng.stream_ptr() if stream is None else C.c_void_p(stream.cuda_stream)
        n = hi - lo
        if n <= 0:
            return
        if self.rows_resampled(lo, hi):
            _check(eng.handle, L.lib().vp_resample(
                eng.handle, C.c_void_p(x.data_ptr()), int(in_ld), C.c_void_p(y.data_ptr()), int(out_ld), n,
                self._ptr(0, 8, lo), self._ptr(1, 8, lo), self._ptr(3, 4, lo), self._ptr(4, 4, lo), self._ptr(2, 8, lo),
                C.c_void_p(eng._taps_dev.data_ptr()), sp))
        if self.gain:
            _check(eng.handle, L.lib().vp_gain_normalize(
                eng.handle, C.c_void_p(y.data_ptr()), int(out_ld), n, self._ptr(1, 8, lo), float(self.target_db),
                self.max_gain_db, C.c_void_p(flags.data_ptr() + 4 * lo), C.c_void_p(scratch.data_ptr()), sp))

    def check(self, flags_host, native_rows=None):
        """Raise AudioSegment.normalize's ValueError for the first flagged row.  The message needs the host's gain:
        it is recomputed from the row's native samples (``native_rows[i]``), resampled and normalised on the host
        exactly as _load_audio did -- an error path only."""
        bad = np.flatnonzero(np.asarray(flags_host))
        if bad.size == 0:
            return
        i = int(bad[0])
        if native_rows is not None:
            from .audio import AudioSegment
            seg = AudioSegment(np.asarray(native_rows[i], dtype=np.float32), int(self.rates[i]))
            seg.resample(self.target_rate)
            seg.normalize(target_db=self.target_db, max_gain_db=self.max_gain_db)      # raises with the host's message
        raise ValueError(f'cannot normalise to {self.target_db} dB: the gain of row {i} exceeds {self.max_gain_db} dB')


class WeightArena:
    """Packs fp32 tensors into one blob; returns byte offsets (256 B aligned)."""

    def __init__(self, chunk_k=1536, kc=512):
        self._chunks = []
        self._size = 0
        self.index = OrderedDict()
        # accumulation-chunk policy of the tensor-core engines (vp_op.tc_kc): layers with K > chunk_k are accumulated in
        # chunks of kc K elements (bounded tensor-core accumulate truncation); deep nets choose shorter values
        self.chunk_k, self.kc = chunk_k, kc

    def add(self, name, arr):
        a = np.ascontiguousarray(np.asarray(arr, dtype=np.float32)).reshape(-1)
        off = self._size
        pad = (-a.nbytes) % ALIGN
        self._chunks.append(a)
        if pad:
            self._chunks.append(np.zeros(pad // 4, dtype=np.float32))
        self._size += a.nbytes + pad
        self.index[name] = (off, a.size)
        return off

    def add_conv(self, name, W2d, tc=True):
        """A conv/linear weight [N, K] (K ordered (tap, ci)): the plain fp32 matrix (exact FFMA engine) plus, for layers
        that can run on the tensor cores, its split-TF32 pre-tiled shared-memory image (conv_tc.cu)."""
        W2d = np.asarray(W2d, dtype=np.float64)
        d = {'w': self.add(name, W2d)}
        if tc and W2d.shape[0] >= 16 and W2d.shape[0] % 4 == 0 and W2d.shape[1] % 4 == 0:
            kc = self.kc if W2d.shape[1] > self.chunk_k else 0
            img, bn = pack_tc(W2d, chunked=kc > 0)
            d['w_tc'] = self.add(name + '.tc', img)
            d['tc_bn'], d['tc_kc'] = bn, kc
            if TC_F16 and W2d.shape[0] >= 128 and W2d.shape[1] >= 8 and W2d.shape[1] % 8 == 0:      # fp16 two-term image (VP_ENGINE_TC16)
                img16, descale = pack_tc16(W2d, bn)
                d['w_tc16'] = self.add(name + '.tc16', img16)
                d['tc16_descale'] = descale
        return d

    def blob(self):
        return np.concatenate(self._chunks) if self._chunks else np.zeros(64, dtype=np.float32)


def tc_tile_n(N, chunked=False):
    """N tile of the tensor-core engine (must match conv_tc.cu::tc_tile_n): the accumulator lives in registers, so tiles
    are 128 wide, except for layers with chunked accumulation (vp_op.tc_kc > 0), which keep a second register set for
    the running sum and therefore use 64-wide tiles."""
    cap = 64 if chunked else 128
    if N >= cap:
        return cap
    return (N + 15) // 16 * 16


def tf32_rna(x):
    """cvt.rna.tf32.f32: round-to-nearest, ties away from zero, to a 10-bit mantissa (fp32 container)."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def pack_tc(W, chunked=None):
    """[N, K] -> (float32 image [n_tiles, k_blocks, 2(hi|lo), BN, 32] with SWIZZLE_128B chunk permutation, BN).
    hi = tf32(W), lo = W - hi (exact in fp32).  Rows >= N / columns >= K are zero.  ``chunked`` (default: K > 1536)
    selects the 64-wide tiles of layers with chunked accumulation."""
    N, K = W.shape
    bn = tc_tile_n(N, K > 1536 if chunked is None else chunked)
    nt, kb = (N + bn - 1) // bn, (K + 31) // 32
    Wp = np.zeros((nt * bn, kb * 32), dtype=np.float32)
    Wp[:N, :K] = W.astype(np.float32)
    hi = tf32_rna(Wp)
    lo = (Wp - hi).astype(np.float32)
    img = np.stack([hi, lo], axis=0).reshape(2, nt, bn, kb, 8, 4)          # [p, nt, r, kb, chunk, 4]
    img = img.transpose(1, 3, 0, 2, 4, 5)                                  # [nt, kb, p, r, chunk, 4]
    r = np.arange(bn)[:, None]
    c = np.arange(8)[None, :]
    out = np.empty_like(img)
    out[:, :, :, r, c ^ (r & 7), :] = img[:, :, :, r, c, :]
    return np.ascontiguousarray(out).reshape(-1), bn


def pack_tc16(W, bn):
    """[N, K] -> (image viewed as float32, descale) for the f16 path of conv_tc.cu.

    The image holds W * 2^k (k chosen so that max|W| 2^k <= 2^14) as two fp16 terms hi = fp16(.), lo = fp16(. - hi),
    tiled [n_tiles, k_blocks of 64, 2 (hi|lo), bn rows, 64 halves] with the 16-byte chunks (8 halves) of every 128-byte
    row XOR-swizzled by (row & 7); descale = 2^-k.  Rows >= N / columns >= K are zero."""
    N, K = W.shape
    nt, kb = (N + bn - 1) // bn, (K + 63) // 64
    wmax = float(np.abs(W).max())
    k = int(np.floor(np.log2(2.0 ** 14 / wmax))) if wmax > 0 else 0
    Wp = np.zeros((nt * bn, kb * 64), dtype=np.float32)
    Wp[:N, :K] = (W * 2.0 ** k).astype(np.float32)
    hi = Wp.astype(np.float16)
    lo = (Wp - hi.astype(np.float32)).astype(np.float16)
    img = np.stack([hi, lo], axis=0).reshape(2, nt, bn, kb, 8, 8)          # [p, nt, r, kb, chunk, 8 halves]
    img = img.transpose(1, 3, 0, 2, 4, 5)                                  # [nt, kb, p, r, chunk, 8]
    r = np.arange(bn)[:, None]
    c = np.arange(8)[None, :]
    out = np.empty_like(img)
    out[:, :, :, r, c ^ (r & 7), :] = img[:, :, :, r, c, :]
    return np.ascontiguousarray(out).reshape(-1).view(np.float32), float(2.0 ** -k)


def unpack_tc16(img, N, K, bn):
    """Inverse of pack_tc16 (tests): -> (hi, lo) float32 [N, K] of the scaled weights."""
    nt, kb = (N + bn - 1) // bn, (K + 63) // 64
    a = np.ascontiguousarray(img).view(np.float16).reshape(nt, kb, 2, bn, 8, 8)
    r = np.arange(bn)[:, None]
    c = np.arange(8)[None, :]
    un = np.empty_like(a)
    un[:, :, :, r, c, :] = a[:, :, :, r, c ^ (r & 7), :]
    un = un.transpose(2, 0, 3, 1, 4, 5).reshape(2, nt * bn, kb * 64).astype(np.float32)
    return un[0, :N, :K], un[1, :N, :K]


class View:
    """A [rows, C] window into an activation buffer: byte offset, row stride (floats), first column, columns.  ``aid`` is
    the planner's allocation id (None for the program input / output and hand-made views): ops that touch the same
    allocation are linked through it when the amax slots of the fp16 split are assigned (PlanBuilder.finalize)."""
    __slots__ = ('off', 'ld', 'coff', 'C', 'aid')

    def __init__(self, off, ld, coff, C_, aid=None):
        self.off, self.ld, self.coff, self.C, self.aid = off, ld, coff, C_, aid

    def cols(self, start, n):
        assert 0 <= start and start + n <= self.C
        return View(self.off, self.ld, self.coff + start, n, self.aid)



class PlanBuilder:
    """Accumulates vp_ops and plans the workspace (first-fit free list: buffers are freed explicitly by the model
    lowering code once their last consumer has been emitted, so big 2-D maps are reused)."""

    def __init__(self, B, engine_pref=L.ENGINE_AUTO):
        self.B = B
        self.ops = []
        self.engine_pref = engine_pref
        self._free = []          # sorted list of [start, end)
        self._top = 0
        self._live = {}
        self.peak = 0
        self.in_floats = 0
        self.out_floats = 0
        self.taps = OrderedDict()   # name -> (View, rows) for tests (vp_program_peek)
        self._next_aid = 0
        self._meta = []             # per op: allocation ids of (dst, src, src2, sum) -- see finalize()
        self._finalized = False

    # ---- memory ----
    def alloc(self, rows, cols):
        nbytes = (rows * cols * 4 + ALIGN - 1) // ALIGN * ALIGN
        for i, (s, e) in enumerate(self._free):
            if e - s >= nbytes:
                if e - s == nbytes:
                    self._free.pop(i)
                else:
                    self._free[i][0] = s + nbytes
                self._live[s] = nbytes
                self._next_aid += 1
                return View(s, cols, 0, cols, self._next_aid)
        s = self._top
        self._top += nbytes
        self.peak = max(self.peak, self._top)
        self._live[s] = nbytes
        self._next_aid += 1
        return View(s, cols, 0, cols, self._next_aid)

    def free(self, view):
        s = view.off
        nbytes = self._live.pop(s)
        self._free.append([s, s + nbytes])
        self._free.sort()
        merged = []
        for iv in self._free:
            if merged and merged[-1][1] == iv[0]:
                merged[-1][1] = iv[1]
            else:
                merged.append(iv)
        if merged and merged[-1][1] == self._top:      # give the tail back
            self._top = merged[-1][0]
            merged.pop()
        self._free = merged

    def input_view(self, cols, rows):
        self.in_floats = rows * cols
        return View(L.BUF_INPUT, cols, 0, cols)

    def input_view1d(self, cols, rows, rows_per_utt):
        """Input of a 1-D (channel = feature) model: CONV gathers float4 along channels, so a feature dim that is not a
        multiple of 4 is first copied into a zero-padded workspace buffer (EW PAD_COPY)."""
        v = self.input_view(cols, rows)
        if cols % 4 == 0:
            return v
        cp = (cols + 3) // 4 * 4
        dst = self.alloc(rows, cp)
        o = self._new(L.OP_EW)
        o.mode = L.EW_PAD_COPY
        o.src, o.in_ld, o.in_coff, o.Cin = v.off, v.ld, v.coff, cols
        o.dst, o.out_ld, o.out_coff, o.Cout = dst.off, dst.ld, dst.coff, cp
        o.Tin, o.Fin = rows_per_utt, 1
        self._emit(o, dst=dst, src=v)
        return dst

    def output_view(self, cols, rows):
        self.out_floats = rows * cols
        return View(L.BUF_OUTPUT, cols, 0, cols)

    def tap(self, name, view, rows):
        self.taps[name] = (view, rows)

    # ---- op emitters ----
    def _new(self, kind):
        o = L.Op()
        o.kind = kind
        o.B = self.B
        for f in ('src', 'src2', 'dst', 'res', 'gate', 'ubias', 'w', 'bias', 'pre_s', 'pre_h', 'post_s', 'post_h', 'w_tc', 'sum'):
            setattr(o, f, -1)
        o.Fin = o.Fout = 1
        o.KT = o.KF = o.sT = o.sF = o.dT = o.dF = 1
        o.seg_len, o.n_seg = 1 << 30, 1
        return o

    def conv(self, src, dst, w, w_ld, Tin, Tout, Fin=1, Fout=1, KT=1, KF=1, sT=1, sF=1, dT=1, dF=1, padT=0, padF=0,
             pad_mode=L.PAD_ZERO, bias=-1, pre=None, pre_relu=False, post=None, act=L.ACT_NONE, act2=L.ACT_NONE,
             res=None, gate=None, ubias=None, seg_len=None, n_seg=1, src2=None, src2_mode=L.SRC2_NONE,
             engine=None, B=None, c1=False, sum_into=None):
        o = self._new(L.OP_CONV_C1 if c1 else L.OP_CONV)
        if B is not None:
            o.B = B
        o.engine = self.engine_pref if engine is None else engine
        o.src, o.in_ld, o.in_coff, o.Cin = src.off, src.ld, src.coff, src.C
        o.dst, o.out_ld, o.out_coff, o.Cout = dst.off, dst.ld, dst.coff, dst.C
        o.Tin, o.Fin, o.Tout, o.Fout = Tin, Fin, Tout, Fout
        o.KT, o.KF, o.sT, o.sF, o.dT, o.dF, o.padT, o.padF, o.pad_mode = KT, KF, sT, sF, dT, dF, padT, padF, pad_mode
        if isinstance(w, dict):            # packed by WeightArena.add_conv: plain + optional tensor-core image
            o.w, o.w_tc, o.tc_bn, o.tc_kc = w['w'], w.get('w_tc', -1), w.get('tc_bn', 0), w.get('tc_kc', 0)
            if 'w_tc16' in w:
                o.w_tc16_q, o.tc16_descale = (w['w_tc16'] >> 4) + 1, w['tc16_descale']
        else:
            o.w = w
        o.w_ld, o.bias = w_ld, bias
        if pre is not None:
            o.pre_s, o.pre_h = pre
            o.pre_relu = 1 if pre_relu else 0
        if post is not None:
            o.post_s, o.post_h = post
        o.act, o.act2 = act, act2
        if res is not None:
            assert res.C == dst.C
            o.res, o.res_ld, o.res_coff = res.off, res.ld, res.coff
        if gate is not None:
            o.gate = gate.off
        if ubias is not None:
            o.ubias = ubias.off
        if seg_len is not None:
            o.seg_len, o.n_seg = seg_len, n_seg
        if src2 is not None:
            o.src2, o.src2_ld, o.src2_coff, o.src2_mode = src2.off, src2.ld, src2.coff, src2_mode
            if src2_mode == L.SRC2_CONCAT:
                o.Cin2 = src2.C
            else:
                assert src2.C == src.C
        if sum_into is not None:           # sum_into[m, :] += y[m, :] after the epilogue (Res2 chains: x_{j+1} += y_j in place)
            assert sum_into.C == dst.C and not c1
            o.sum, o.sum_ld, o.sum_coff = sum_into.off, sum_into.ld, sum_into.coff
        self._check_conv(o)
        self._emit(o, dst=dst, src=src, src2=src2, summed=sum_into)
        return o

    @staticmethod
    def _check_conv(o):
        """Same alignment rules the C validator enforces (api.cu validate_op), raised early on the host."""
        def a4(*vals):
            return all(v % 4 == 0 for v in vals)
        if o.kind == L.OP_CONV_C1:
            ok = o.Cin == 1 and a4(o.Cout, o.out_ld, o.out_coff)
        else:
            ok = a4(o.Cin, o.in_ld, o.in_coff, o.w_ld, o.Cin2)
            if o.src2_mode != L.SRC2_NONE:
                ok = ok and a4(o.src2_ld, o.src2_coff)
        if not ok:
            raise ValueError('conv op: channel counts / strides / offsets must be multiples of 4 floats '
                             f'(Cin={o.Cin}, Cin2={o.Cin2}, in_ld={o.in_ld}, in_coff={o.in_coff}, w_ld={o.w_ld})')

    def colstats(self, src, dst, rows_per_utt, mode, eps=0.0, seg_len=None, n_seg=1):
        o = self._new(L.OP_COLSTATS)
        o.mode = mode
        o.src, o.in_ld, o.in_coff, o.Cin = src.off, src.ld, src.coff, src.C
        o.dst, o.out_ld, o.out_coff = dst.off, dst.ld, dst.coff
        o.Tin, o.Fin = rows_per_utt, 1
        o.eps = eps
        if seg_len is not None:
            o.seg_len, o.n_seg = seg_len, n_seg
        self._emit(o, dst=dst, untracked=True)
        return o

    def asp_pool(self, x, logits, dst, T, eps=1e-12, mean_only=False):
        o = self._new(L.OP_ASP_POOL)
        o.mode = 1 if mean_only else 0
        o.src, o.in_ld, o.in_coff, o.Cin = x.off, x.ld, x.coff, x.C
        o.src2, o.src2_ld, o.src2_coff = logits.off, logits.ld, logits.coff
        o.dst, o.out_ld, o.out_coff = dst.off, dst.ld, dst.coff
        o.Tin = T
        o.eps = eps
        self._emit(o, dst=dst, untracked=True)
        return o

    def pool2d(self, src, dst, mode, Tin, Fin, Tout, Fout, k=3, stride=1, pad=1):
        o = self._new(L.OP_POOL2D)
        o.mode = mode
        o.src, o.in_ld, o.in_coff, o.Cin = src.off, src.ld, src.coff, src.C
        o.dst, o.out_ld, o.out_coff = dst.off, dst.ld, dst.coff
        o.Tin, o.Fin, o.Tout, o.Fout = Tin, Fin, Tout, Fout
        o.KT = o.KF = k
        o.sT = o.sF = stride
        o.padT = o.padF = pad
        self._emit(o, dst=dst, src=src)
        return o

    def ew(self, mode, x, dst, rows_per_utt, gate=None, res=None, y=None, att=None, act2=L.ACT_NONE):
        o = self._new(L.OP_EW)
        o.mode = mode
        o.src, o.in_ld, o.in_coff, o.Cin = x.off, x.ld, x.coff, x.C
        o.dst, o.out_ld, o.out_coff = dst.off, dst.ld, dst.coff
        o.Tin, o.Fin = rows_per_utt, 1
        o.act2 = act2
        if gate is not None:
            o.gate = gate.off
        if res is not None:
            o.res, o.res_ld, o.res_coff = res.off, res.ld, res.coff
        if y is not None:
            o.src2, o.src2_ld, o.src2_coff = y.off, y.ld, y.coff
        if att is not None:
            o.res, o.res_ld, o.res_coff = att.off, att.ld, att.coff
        self._emit(o, dst=dst, src=x)
        return o

    # ---- amax slots of the fp16 split (include/vpb200.h: vp_op.amax_out / amax_in) ----
    def _emit(self, o, dst=None, src=None, src2=None, summed=None, untracked=False):
        aid = lambda v: getattr(v, 'aid', None) if v is not None else None
        self._meta.append(dict(dst=aid(dst), src=aid(src), src2=aid(src2), summed=aid(summed), untracked=untracked))
        self.ops.append(o)
        self._finalized = False

    def finalize(self):
        """Assign amax slots: one slot per workspace allocation that a CONV with an fp16 weight image reads as its
        (whole) source; every op writing into that allocation maxes |y| into the slot, the CONV scales by it.  An
        allocation written by an op that does not track amax (pooling kernels, accumulate-into views) gets no slot, so
        its consumers stay on split TF32.  Idempotent."""
        if self._finalized:
            return self
        for o in self.ops:
            o.amax_out = o.amax_in = 0
        bad = set()
        for o, m in zip(self.ops, self._meta):
            if m['untracked'] and m['dst'] is not None:
                bad.add(m['dst'])
            if m['summed'] is not None:
                bad.add(m['summed'])
        slots = {}
        for o, m in zip(self.ops, self._meta):
            if o.kind != L.OP_CONV or o.w_tc16_q <= 0 or m['src'] is None or m['src'] in bad:
                continue
            if o.pre_s >= 0 or o.src2_mode == L.SRC2_ADD:
                continue                                    # source modes the fp16 kernel does not implement
            if o.src2_mode == L.SRC2_CONCAT and m['src2'] != m['src']:
                continue                                    # two tensors, one scale: only when they share an allocation
            o.amax_in = slots.setdefault(m['src'], len(slots)) + 1
        for o, m in zip(self.ops, self._meta):
            if m['dst'] in slots:
                o.amax_out = slots[m['dst']] + 1
        self._finalized = True
        return self


class Program:
    """A compiled (validated, workspace-backed) program for one (B, T)."""

    def __init__(self, engine, pb):
        self.engine = engine
        self.n_ops = len(pb.ops)
        self.ws_bytes = max(pb.peak, ALIGN)
        self.in_floats, self.out_floats = pb.in_floats, pb.out_floats
        self.taps = pb.taps
        pb.finalize()
        arr = (L.Op * self.n_ops)(*pb.ops)
        self._p = C.c_void_p()
        _check(engine.handle, L.lib().vp_program_create(engine.handle, arr, self.n_ops, self.ws_bytes,
                                                        self.in_floats, self.out_floats, C.byref(self._p)))
        engine._programs.append(self)

    @property
    def launches(self):
        return int(L.lib().vp_program_launches(self._p))

    def run(self, feats, emb):
        assert feats.is_cuda and feats.dtype == torch.float32 and feats.is_contiguous()
        assert emb.is_cuda and emb.dtype == torch.float32 and emb.is_contiguous()
        assert feats.numel() == self.in_floats and emb.numel() == self.out_floats
        _check(self.engine.handle, L.lib().vp_embed(self._p, C.c_void_p(feats.data_ptr()), C.c_void_p(emb.data_ptr()),
                                                    self.engine.stream_ptr()))

    def run_profiled(self, feats, emb):
        """vp_embed with per-op CUDA-event timing -> list of dicts (kind, M, N, K, engine, ms)."""
        ms = (C.c_float * self.n_ops)()
        _check(self.engine.handle, L.lib().vp_embed_profiled(self._p, C.c_void_p(feats.data_ptr()),
                                                             C.c_void_p(emb.data_ptr()), self.engine.stream_ptr(), ms))
        out = []
        for i in range(self.n_ops):
            kind, eng = C.c_int32(), C.c_int32()
            M, N, K = C.c_int64(), C.c_int64(), C.c_int64()
            L.lib().vp_program_op_info(self._p, i, C.byref(kind), C.byref(M), C.byref(N), C.byref(K), C.byref(eng))
            out.append(dict(op=i, kind=kind.value, M=M.value, N=N.value, K=K.value, engine=eng.value, ms=float(ms[i])))
        return out

    def peek(self, name):
        """Copy a tapped intermediate out of the workspace (tests only)."""
        view, rows = self.taps[name]
        n = (rows - 1) * view.ld + view.coff + view.C
        buf = torch.empty(n, dtype=torch.float32, device=self.engine.device)
        _check(self.engine.handle, L.lib().vp_program_peek(self._p, view.off, n * 4, C.c_void_p(buf.data_ptr()),
                                                           self.engine.stream_ptr()))
        full = torch.zeros(rows * view.ld, dtype=torch.float32, device=self.engine.device)
        full[:n] = buf
        return full.view(rows, view.ld)[:, view.coff:view.coff + view.C]

    def close(self):
        if self._p:
            L.lib().vp_program_destroy(self._p)
            self._p = C.c_void_p()
            try:
                self.engine._programs.remove(self)       # a long-lived server must not accumulate closed programs
            except ValueError:
                pass
