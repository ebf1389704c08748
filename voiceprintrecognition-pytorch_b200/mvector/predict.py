"""MVectorPredictor: drop-in for mvector.predict.MVectorPredictor (reference: mvector/predict.py:22-395) on the
GPU-native path.  Constructor and method signatures, argument meaning and error behaviour follow the reference;
``predict`` / ``predict_batch`` / ``contrast`` run entirely on hand-written sm_90a kernels through libvpb200.so.

Differences that are deliberate:
  * ``use_gpu=False`` raises: this path has no CPU implementation (the reference's CPU path is the oracle).
  * ``predict_batch`` feeds the WHOLE padded batch to the device in one ``vp_embed_wave`` call (front-end + backbone);
    the reference's ``batch_size`` argument (predict.py:261) is accepted and ignored -- chunking does not change
    results because every op is per-utterance, and padding/CMN/mask are computed on the full batch exactly like
    predict.py:244-258.
  * ``speaker_diarization`` (predict.py:365-395): chunk embeddings come from ``predict_batch`` on the device, and
    so does the spectral stage of the clustering up to its eigenvectors (``Engine.spectral_embedding``); chunking,
    k-means and post-processing are host glue (infer_utils/speaker_diarization.py); the VAD is an energy
    detector standing in for yeaudio's model-based one (absent third-party code, outside the parity boundary).
"""
import os
import pickle
import shutil
from io import BufferedReader

import numpy as np
import torch
import yaml
from loguru import logger

from .audio import AudioSegment
from .data_utils.featurizer import AudioFeaturizer
from .engine import Engine
from .infer_utils.speaker_diarization import SpeakerDiarization
from .models import build_model
from .utils.checkpoint import load_pretrained
from .utils.utils import dict_to_object, print_arguments


class MVectorPredictor:
    def __init__(self, configs, threshold=0.6, audio_db_path=None, model_path='models/CAMPPlus_Fbank/best_model/',
                 use_gpu=True):
        if use_gpu:
            assert torch.cuda.is_available(), 'GPU不可用'
            self.device = torch.device('cuda', torch.cuda.current_device())
        else:
            raise RuntimeError('use_gpu=False: the GPU-native path has no CPU implementation')
        self.threshold = threshold
        if isinstance(configs, str):
            with open(configs, 'r', encoding='utf-8') as f:
                configs = yaml.load(f.read(), Loader=yaml.FullLoader)
            print_arguments(configs=configs)
        self.configs = dict_to_object(configs)
        self._engine = Engine(self.device.index)
        self._audio_featurizer = AudioFeaturizer(feature_method=self.configs.preprocess_conf.feature_method,
                                                 use_hf_model=self.configs.preprocess_conf.get('use_hf_model', False),
                                                 method_args=self.configs.preprocess_conf.get('method_args', {}),
                                                 engine=self._engine)
        self.predictor = build_model(input_size=self._audio_featurizer.feature_dim, configs=self.configs)
        self.predictor.engine = self._engine
        if os.path.isdir(model_path):
            model_path = os.path.join(model_path, 'model.pth')
        assert os.path.exists(model_path), f"{model_path} 模型不存在！"
        self.predictor = load_pretrained(self.predictor, model_path, use_gpu=use_gpu)
        logger.info(f"成功加载模型参数：{model_path}")
        self.predictor.eval()
        self._pinned = None
        self._copy_stream = None
        self._ws_per_utt = {}
        self._trace = None
        self._trace_dev = None

        self.speaker_diarize = SpeakerDiarization()
        # spectral stage of the clustering (speaker_diarization.py:244-248: affinity, pruning, Laplacian, eigenvectors)
        # on the device
        self.speaker_diarize.set_spectral(self._engine.spectral_embedding)

        self.audio_feature = None
        self.audio_feature_mean = None
        self.users_name = []
        self.users_audio_path = []
        self.users_name_mean = []
        self.audio_db_path = audio_db_path
        if self.audio_db_path is not None:
            self.audio_indexes_path = os.path.join(audio_db_path, "audio_indexes.bin")
            self.__load_audio_db(self.audio_db_path)

    # ------------------------------------------------------------------ voiceprint DB (numpy glue, predict.py:85-183)
    def __load_audio_indexes(self):
        if not os.path.exists(self.audio_indexes_path):
            return
        with open(self.audio_indexes_path, "rb") as f:
            indexes = pickle.load(f)
        for name, feature, path in zip(indexes["users_name"], indexes["faces_feature"], indexes["users_image_path"]):
            if not os.path.exists(path):
                continue
            self.users_name.append(name)
            self.users_audio_path.append(path)
            self.audio_feature = feature if self.audio_feature is None else np.vstack((self.audio_feature, feature))

    def __write_index(self):
        with open(self.audio_indexes_path, "wb") as f:
            pickle.dump({"users_name": self.users_name, "faces_feature": self.audio_feature,
                         "users_image_path": self.users_audio_path}, f)

    def __refresh_means(self):
        self.audio_feature_mean, self.users_name_mean = None, []
        for name in set(self.users_name):
            idx = [i for i, v in enumerate(self.users_name) if v == name]
            feature = self.audio_feature[idx].mean(axis=0)
            self.audio_feature_mean = feature if self.audio_feature_mean is None \
                else np.vstack((self.audio_feature_mean, feature))
            self.users_name_mean.append(name)
        if self.audio_feature_mean is not None and len(self.audio_feature_mean.shape) == 1:
            self.audio_feature_mean = self.audio_feature_mean[np.newaxis, :]

    def __load_audio_db(self, audio_db_path):
        self.__load_audio_indexes()
        os.makedirs(audio_db_path, exist_ok=True)
        paths = []
        for name in os.listdir(audio_db_path):
            d = os.path.join(audio_db_path, name)
            if not os.path.isdir(d):
                continue
            for file in os.listdir(d):
                paths.append(os.path.join(d, file).replace('\\', '/'))
        if len(paths) == 0:
            return
        logger.info('正在加载声纹库数据...')
        bs = self.configs.dataset_conf.eval_conf.batch_size
        pending = []
        for p in paths:
            if p in self.users_audio_path:
                continue
            seg = self._load_audio(p)
            self.users_name.append(os.path.basename(os.path.dirname(p)))
            self.users_audio_path.append(p)
            pending.append(seg)                       # at its own rate: conditioned on the device by predict_batch
            if len(pending) == bs:
                feats = self.predict_batch(pending)
                self.audio_feature = feats if self.audio_feature is None else np.vstack((self.audio_feature, feats))
                pending = []
        if pending:
            feats = self.predict_batch(pending)
            self.audio_feature = feats if self.audio_feature is None else np.vstack((self.audio_feature, feats))
        assert len(self.audio_feature) == len(self.users_name) == len(self.users_audio_path), '加载的数量对不上！'
        self.__write_index()
        self.__refresh_means()
        logger.info(f'声纹库数据加载完成，一共有{len(self.audio_feature_mean)}个用户，分别是：{self.users_name_mean}')

    @staticmethod
    def normalize_features(features):
        return features / np.linalg.norm(features, axis=1, keepdims=True)

    def __retrieval(self, np_feature):
        if isinstance(np_feature, list):
            np_feature = np.array(np_feature)
        sims = self._engine.cosine_scores(np_feature.astype(np.float32), self.audio_feature_mean).cpu().numpy()
        labels = []
        for sim in sims:                                       # cosine similarity on the device (predict.py:169-183)
            idx = int(np.argmax(sim))
            s = sim[idx]
            labels.append([self.users_name_mean[idx], round(float(s), 5)] if s >= self.threshold else [None, None])
        return labels

    # ------------------------------------------------------------------ hot path
    def _load_audio(self, audio_data, sample_rate=16000):
        """predict.py:185-204: decoding, type dispatch and the min-duration assert on the NATIVE duration -> the
        AudioSegment at its own rate.  Resampling and dB normalisation (predict.py:205-211) run on the device, in the
        staging of ``_embed_waves``; ``_condition_host`` is the host form for the callers that need host samples."""
        if isinstance(audio_data, str):
            audio_segment = AudioSegment.from_file(audio_data)
        elif isinstance(audio_data, BufferedReader):
            audio_segment = AudioSegment.from_file(audio_data)
        elif isinstance(audio_data, np.ndarray):
            audio_segment = AudioSegment.from_ndarray(audio_data, sample_rate)
        elif isinstance(audio_data, bytes):
            audio_segment = AudioSegment.from_bytes(audio_data)
        elif isinstance(audio_data, AudioSegment):
            audio_segment = audio_data
        else:
            raise Exception(f'不支持该数据类型，当前数据类型为：{type(audio_data)}')
        ds = self.configs.dataset_conf.dataset
        assert audio_segment.duration >= ds.min_duration, \
            f'音频太短，最小应该为{ds.min_duration}s，当前音频为{audio_segment.duration}s'
        return audio_segment

    def _condition_host(self, audio_segment):
        """predict.py:205-211 on the host, in place: ``register`` writes the normalised samples to disk and
        ``speaker_diarization`` runs its VAD on them."""
        ds = self.configs.dataset_conf.dataset
        if audio_segment.sample_rate != ds.sample_rate:
            audio_segment.resample(ds.sample_rate)
        if ds.use_dB_normalization:
            audio_segment.normalize(target_db=ds.target_dB)
        return audio_segment

    #: utterances per backbone program (one fused vp_embed per chunk); the workspace limit can lower it for big 2-D nets
    MAX_BATCH = 256
    #: utterances per staging call (host gather -> pinned -> H2D -> front-end kernels), double buffered
    STAGE_ROWS = 128
    #: utterances per H2D copy inside a staging call (the copy of slice k overlaps the gather of slice k+1)
    COPY_SLICE = 4
    #: utterances per backbone program on the HOST-staged path: smaller than MAX_BATCH so that the backbone of chunk k runs
    #: while the host gathers and copies chunk k+1
    HOST_CHUNK = 128
    _gather_configured = False
    #: program workspace cap: leaves an 80 GB H100 room for weights, inputs and the caller's own tensors
    WS_LIMIT_BYTES = int(float(os.environ.get('VPB_WS_LIMIT_GB', '48')) * 2 ** 30)

    @classmethod
    def _configure_gather(cls, lib):
        """Staging gather with non-temporal stores only when several ranks share this host: their gathers run at the same
        time and are DRAM-bound, while the single-process path keeps the measured memcpy gather."""
        if not cls._gather_configured:
            on = int(os.environ.get('LOCAL_WORLD_SIZE', '1')) > 1
            lib.vp_host_gather_streaming(1 if on else 0)
            cls._gather_configured = True

    @staticmethod
    def _gather_threads():
        """Host threads of the staging gather: what this process may use, split between the ranks of the node."""
        if os.environ.get('VPB_GATHER_THREADS'):
            return max(1, int(os.environ['VPB_GATHER_THREADS']))
        try:
            ncpu = len(os.sched_getaffinity(0))
        except AttributeError:
            ncpu = os.cpu_count() or 1
        local_world = max(1, int(os.environ.get('LOCAL_WORLD_SIZE', '1')))
        if ncpu < (os.cpu_count() or ncpu):
            local_world = 1          # the launcher already gave this rank its own CPU slice (bind_rank_to_local_cpus)
        per_rank = ncpu // local_world
        quota = MVectorPredictor._cgroup_cpus()
        if quota is not None:
            # a container CPU quota is shared by ALL ranks of the node, bound or not.  Under CFS bandwidth control every
            # short-lived wake-up of a worker thread also strands up to 1 ms of quota on its core, so many threads per rank
            # get the whole job throttled: never more threads than this rank's share
            per_rank = min(per_rank, int(quota // max(1, int(os.environ.get('LOCAL_WORLD_SIZE', '1')))))
        return max(1, min(8, per_rank))                 # the calling thread counts: it gathers between issuing copies

    _quota_cache = []

    @staticmethod
    def _cgroup_cpus():
        """CPUs' worth of time the container may use (cgroup v2 cpu.max / v1 cfs quota), or None when unlimited."""
        if not MVectorPredictor._quota_cache:
            MVectorPredictor._quota_cache.append(MVectorPredictor._read_cgroup_cpus())
        return MVectorPredictor._quota_cache[0]

    @staticmethod
    def _read_cgroup_cpus():
        try:
            with open('/sys/fs/cgroup/cpu.max') as f:
                q, p = f.read().split()
            return None if q == 'max' else float(q) / float(p)
        except Exception:
            pass
        try:
            with open('/sys/fs/cgroup/cpu/cpu.cfs_quota_us') as f:
                q = float(f.read())
            with open('/sys/fs/cgroup/cpu/cpu.cfs_period_us') as f:
                p = float(f.read())
            return None if q <= 0 else q / p
        except Exception:
            return None

    def _pinned_slot(self, slot, n):
        """Two reusable pinned host staging buffers (double buffering)."""
        if self._pinned is None:
            self._pinned = [None, None]
        if self._pinned[slot] is None or self._pinned[slot].numel() < n:
            self._pinned[slot] = torch.empty(max(n, 1 << 20), dtype=torch.float32).pin_memory()
        return self._pinned[slot][:n]

    def _chunk_size(self, B, T):
        """Utterances per backbone program: MAX_BATCH, lowered so that the program workspace stays under WS_LIMIT_BYTES
        (ERes2Net-55M at T = 998 needs ~0.6 GB per utterance)."""
        cb = min(self.MAX_BATCH, B)
        per = self._ws_per_utt.get(T)
        if per is None:
            per = self._ws_per_utt[T] = max(int(self.predictor.lower(1, T).peak), 1)
        return max(1, min(cb, self.WS_LIMIT_BYTES // per))

    def _host_chunks(self, B, T):
        """Backbone chunk sizes of the host-staged path: about HOST_CHUNK utterances each (never above ``_chunk_size``), the
        cut placed -- within 8 utterances -- where the chunk's row count fills whole waves of 128-row tiles on the 132 SMs of
        an H100 (at T = 275, 122 utterances are 263 tiles = two waves, 123 utterances spill into a third)."""
        limit = min(self._chunk_size(B, T), max(self.HOST_CHUNK, 1))
        sms = 132

        def waste(c):
            tiles = -(-c * T // 128)
            return (-(-tiles // sms) * sms - tiles) / float(-(-tiles // sms) * sms)
        out, left = [], B
        while left > 0:
            if left <= limit + 8 and left <= self._chunk_size(B, T):
                out.append(left)
                break
            c = min(range(max(limit - 8, 1), limit + 1), key=lambda n: (round(waste(n), 3), -n))
            out.append(c)
            left -= c
        return out

    def _embed_waves(self, waves, lmax, masked, to_numpy=True, group=None, rates=None):
        """waves: list of 1-D float32 arrays, decoded, at ``rates`` Hz (None: all at the model's rate) -> [B, embd_dim]
        (np.float32, or the device tensor with ``to_numpy=False``).  ``lmax`` is the longest item AFTER resampling.

        Conditioning (predict.py:205-211) runs on the device inside the staging: a stage with rows to resample is
        gathered at its native length into a native-rate device slot and resampled into the model-rate slot
        (vp_resample); with ``use_dB_normalization`` the rows are then normalised in place (vp_gain_normalize), before
        the front-end.  A gain above 300 dB raises ValueError before the call returns.  A call that needs neither
        enqueues nothing of the two.

        Reference semantics (predict.py:244-262): every utterance is zero padded to ``lmax`` (the longest item of the WHOLE
        batch -- the caller's batch, which under ``predict_batch_sharded`` is larger than this rank's list), T and the CMN
        mean follow that padded length, frames >= round(len/Lmax * T) are zeroed.

        Pipeline (every op is per-utterance, so slicing the batch cannot change results): staging calls of STAGE_ROWS
        utterances -- native threads gather them into pinned memory and the H2D copies are issued on the copy stream as
        slices finish (``vp_host_stage_h2d``) -- feed the fused front-end kernels, which run on the main stream behind an
        event of their stage's copies and write straight into the [B, T, F] feature buffer; as soon as the features of a
        backbone chunk (``_host_chunks``) are complete the main stream runs its program, under the next stage's gather and
        copies.  One D2H of the result at the end."""
        from . import _lib as L
        import ctypes as C
        import time
        tr = self._trace                                 # None, or a list the caller wants (label, perf_counter) pairs in
        mark = (lambda label: tr.append((label, time.perf_counter()))) if tr is not None else (lambda label: None)
        mark('embed_waves:start')
        B = len(waves)
        fz = self._audio_featurizer
        D = self.predictor.embd_dim
        dev = self.device
        if B == 0:
            e = torch.empty(0, D, dtype=torch.float32, device=dev)
            return e.cpu().numpy() if to_numpy else e
        T = fz.num_frames(lmax)
        desc = fz.feat_fun.desc
        if desc.kind == 0:
            assert 2 <= fz.feat_fun.win_length <= lmax, f'choose a window size {fz.feat_fun.win_length} that is [2, {lmax}]'
        eng = fz.engine
        lib = L.lib()
        F = fz.feature_dim
        ds_conf = self.configs.dataset_conf.dataset
        lens = np.fromiter(map(len, waves), dtype=np.int32, count=B)
        plan = None
        gain_db = ds_conf.target_dB if ds_conf.use_dB_normalization else None
        if gain_db is not None or (rates is not None and any(int(r) != ds_conf.sample_rate for r in rates)):
            plan = eng.condition_plan(lens, ds_conf.sample_rate if rates is None else rates, ds_conf.sample_rate, gain_db)
        keep_all = None
        if masked:
            lens64 = plan.n_out if plan is not None else lens.astype(np.int64)
            # float64 quotient rounded once to float32 == torch.tensor([len / lmax ...], dtype=float32) of predict.py:251-255
            keep_all = fz.keep_frames(torch.from_numpy((lens64 / lmax).astype(np.float32)), T).to(dev)
        emb = torch.empty(B, D, dtype=torch.float32, device=dev)
        feats = torch.empty(B, T * F, dtype=torch.float32, device=dev)
        bounds = np.cumsum(self._host_chunks(B, T)).tolist()       # end row of every backbone chunk
        whole = desc.post == 1 and desc.top_db >= 0      # MFCC: the top_db clamp needs the maximum over the whole call
        S = B if whole else min(self.STAGE_ROWS, B)
        nstages = (B + S - 1) // S
        K = min(nstages, 4)                             # device staging slots (the pinned side always has two)
        dwave = torch.empty(K, S * lmax, dtype=torch.float32, device=dev)
        dnat = flags = gscratch = None
        if plan is not None:
            if plan.resample:                            # native-rate slots of the stages that resample
                dnat = torch.empty(K, S * int(lens.max()), dtype=torch.float32, device=dev)
            if plan.gain:
                flags = torch.empty(B, dtype=torch.int32, device=dev)
                gscratch = plan.scratch(S, lmax)
        scratch = torch.empty(max(int(lib.vp_frontend_scratch_floats(eng.handle, S, lmax)), 1), dtype=torch.float32, device=dev)
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=dev)
        cs = self._copy_stream
        cs_ptr = C.c_void_p(cs.cuda_stream)
        main = torch.cuda.current_stream(dev)
        main_ptr = C.c_void_p(main.cuda_stream)
        cs.wait_stream(main)                            # buffers handed out by the allocator may still be in use on main
        ptrs = np.empty(B, dtype=np.uint64)              # filled stage by stage: only stage 0's part is on the critical path
        nthreads = self._gather_threads()
        self._configure_gather(lib)
        mark('host prep done (keep, buffers, pointer table)')
        dtr = self._trace_dev                           # None, or a list for (label, timing event) pairs

        def dmark(label, stream):
            if dtr is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record(stream)
                dtr.append((label, e))
        dmark('t0 (main stream)', main)
        fe_fn = lib.vp_fbank if desc.kind == 0 else (lib.vp_mfcc if desc.post == 1 else lib.vp_melspec)
        pin_ev = [None, None]                           # H2D copies out of a pinned slot finished: the host may refill it
        dev_ev = [None] * K                             # front-end finished reading a device slot: the copies may refill it
        next_chunk = 0
        for gi, g0 in enumerate(range(0, B, S)):
            g1 = min(g0 + S, B)
            n = g1 - g0
            ps, ds = gi & 1, gi % K
            if pin_ev[ps] is not None:
                pin_ev[ps].synchronize()
            if dev_ev[ds] is not None:
                cs.wait_event(dev_ev[ds])
            dw = dwave[ds]
            resample = plan is not None and plan.rows_resampled(g0, g1)
            ld = int(lens[g0:g1].max()) if resample else lmax          # a resampling stage stages its native rows
            dst = dnat[ds] if resample else dw
            host = self._pinned_slot(ps, n * ld)
            ptrs[g0:g1] = np.fromiter((w.__array_interface__['data'][0] for w in waves[g0:g1]), dtype=np.uint64, count=n)
            rc = lib.vp_host_stage_h2d(C.c_void_p(ptrs.ctypes.data + 8 * g0), C.c_void_p(lens.ctypes.data + 4 * g0), n, ld,
                                       C.c_void_p(host.data_ptr()), C.c_void_p(dst.data_ptr()), self.COPY_SLICE, nthreads, cs_ptr)
            if rc != L.VP_OK:
                raise L.VpError(rc, 'vp_host_stage_h2d failed')
            mark(f'stage {gi}: {n} utterances gathered, H2D enqueued')
            cev = torch.cuda.Event()
            cev.record(cs)
            pin_ev[ps] = cev
            dmark(f'stage {gi}: H2D done', cs)
            main.wait_event(cev)
            if plan is not None:
                plan.run(dst, ld, dw, lmax, g0, g1, flags, gscratch, main)
                dmark(f'stage {gi}: conditioning done', main)
            kp = C.c_void_p(keep_all.data_ptr() + 4 * g0) if keep_all is not None else C.c_void_p()
            if whole and group is not None:
                fz.mfcc_sharded(dw, n, lmax, kp, feats, scratch, main, group)
            else:
                from .engine import _check
                _check(eng.handle, fe_fn(eng.handle, C.c_void_p(dw.data_ptr()), n, lmax, kp,
                                         C.c_void_p(feats.data_ptr() + 4 * g0 * T * F), C.c_void_p(scratch.data_ptr()), main_ptr))
            fev = torch.cuda.Event()
            fev.record(main)
            dev_ev[ds] = fev
            dmark(f'stage {gi}: front-end done', main)
            # backbone chunks whose features are now complete
            while bounds and bounds[0] <= g1:
                hi = bounds.pop(0)
                self.predictor.program(hi - next_chunk, T).run(feats[next_chunk:hi], emb[next_chunk:hi])
                dmark(f'backbone rows {next_chunk}:{hi} done', main)
                next_chunk = hi
        # the staging / feature buffers go back to the allocator for the main stream: order the copy stream before that
        main.wait_stream(cs)
        mark('all kernels enqueued')
        out = emb.cpu().numpy() if to_numpy else emb
        if flags is not None:
            plan.check(flags.cpu().numpy(), waves)      # after the result copy: no extra synchronise
        mark('result on host' if to_numpy else 'returned device tensor')
        return out

    def embed_device(self, wave_dev, lens=None, lmax=None, keep=None, group=None, out=None):
        """Device-resident twin of ``predict_batch``'s compute half: ``wave_dev`` is a CUDA float32 ``[B, Lmax]`` matrix,
        zero padded to the longest item of the (global) batch; ``lens`` the true sample counts (None: every row is full
        length, i.e. no masking) or ``keep`` the precomputed device int32 mask lengths.  Returns the device tensor
        ``[B, embd_dim]`` (``out`` when given: a contiguous CUDA float32 ``[B, embd_dim]`` view to write into).  One fused
        ``vp_embed_wave`` (front-end + backbone) per chunk of <= MAX_BATCH utterances; nothing is copied or synchronised."""
        from . import _lib as L
        assert wave_dev.is_cuda and wave_dev.dtype == torch.float32 and wave_dev.dim() == 2 and wave_dev.is_contiguous()
        B, Lp = wave_dev.shape
        assert lmax is None or lmax == Lp
        fz = self._audio_featurizer
        T = fz.num_frames(Lp)
        desc = fz.feat_fun.desc
        if keep is None and lens is not None:
            keep = fz.keep_frames(torch.tensor([n / Lp for n in lens], dtype=torch.float32), T).to(wave_dev.device)
        D, F = self.predictor.embd_dim, fz.feature_dim
        if out is not None:
            assert out.is_cuda and out.dtype == torch.float32 and tuple(out.shape) == (B, D) and out.is_contiguous()
        emb = out if out is not None else torch.empty(B, D, dtype=torch.float32, device=wave_dev.device)
        cb = self._chunk_size(B, T)
        if desc.post == 1 and desc.top_db >= 0:         # MFCC: call-wide clamp -> front-end on the whole batch first
            feats = fz.forward_keep(wave_dev, keep, group=group)
            for lo in range(0, B, cb):
                hi = min(lo + cb, B)
                self.predictor.program(hi - lo, T).run(feats[lo:hi].contiguous(), emb[lo:hi])
            return emb
        eng = fz.engine
        feats = torch.empty(cb * T * F, dtype=torch.float32, device=wave_dev.device)
        scratch = torch.empty(max(int(L.lib().vp_frontend_scratch_floats(eng.handle, cb, Lp)), 1), dtype=torch.float32,
                              device=wave_dev.device)
        for lo in range(0, B, cb):
            hi = min(lo + cb, B)
            self.predictor.program(hi - lo, T).run_wave(wave_dev[lo:hi], None if keep is None else keep[lo:hi],
                                                        feats[:(hi - lo) * T * F], scratch, emb[lo:hi])
        return emb

    def predict(self, audio_data, sample_rate=16000):
        """预测一个音频的特征 (predict.py:214-229) -> np.ndarray [embd_dim]"""
        seg = self._load_audio(audio_data=audio_data, sample_rate=sample_rate)
        w = np.ascontiguousarray(seg.samples, dtype=np.float32)
        lmax = int(self._output_lengths([w.shape[0]], [seg.sample_rate])[0])
        return self._embed_waves([w], lmax, masked=False, rates=[seg.sample_rate])[0]

    def predict_batch(self, audios_data, sample_rate=16000, batch_size=32):
        """预测一批音频的特征 (predict.py:231-265) -> np.ndarray [B, embd_dim], order preserved."""
        waves, rates = self._load_batch(audios_data, sample_rate)
        lmax = int(self._output_lengths(list(map(len, waves)), rates).max()) if waves else 0
        return self._embed_waves(waves, lmax, masked=True, rates=rates)

    def _output_lengths(self, n_in, rates):
        """Sample counts after resampling to the model's rate (int64 numpy): known on the host before anything runs."""
        from .audio import resample_ratio, resampled_length
        tsr = self.configs.dataset_conf.dataset.sample_rate
        ratio = {r: resample_ratio(r, tsr) for r in set(rates)}
        return resampled_length(n_in, [ratio[r][0] for r in rates], [ratio[r][1] for r in rates])

    def _load_batch(self, audios_data, sample_rate=16000):
        """predict.py:244-247 for a list -> (decoded float32 rows at their native rate, the rates).  C-contiguous float32
        1-D arrays come out of ``_load_audio`` unchanged (predict.py:196-204: from_ndarray, duration assert) -- they are
        checked in one pass and used in place instead of being wrapped one by one (a 256-utterance batch spends more time
        in that loop than the GPU in its front-end); resampling and normalisation follow on the device."""
        ds = self.configs.dataset_conf.dataset
        if all(type(a) is np.ndarray and a.dtype == np.float32 and a.ndim == 1 and a.flags.c_contiguous for a in audios_data):
            shortest = min(a.shape[0] for a in audios_data) if len(audios_data) else 0
            if len(audios_data) == 0 or shortest / float(sample_rate) >= ds.min_duration:
                return list(audios_data), [int(sample_rate)] * len(audios_data)
        segs = [self._load_audio(audio_data=a, sample_rate=sample_rate) for a in audios_data]
        return [np.ascontiguousarray(s.samples, dtype=np.float32) for s in segs], [s.sample_rate for s in segs]

    def contrast(self, audio_data1, audio_data2):
        """声纹对比 (predict.py:267-279) -> cosine similarity"""
        f1 = self.predict(audio_data1)
        f2 = self.predict(audio_data2)
        return np.dot(f1, f2) / (np.linalg.norm(f1) * np.linalg.norm(f2))

    def register(self, audio_data, user_name: str, sample_rate=16000):
        """声纹注册 (predict.py:281-309)"""
        seg = self._condition_host(self._load_audio(audio_data=audio_data, sample_rate=sample_rate))
        feature = self.predict(audio_data=seg.samples, sample_rate=seg.sample_rate)
        if self.audio_feature is None:
            self.audio_feature = feature
        else:
            self.audio_feature = np.vstack((self.audio_feature, feature))
        if self.audio_feature.ndim == 1:
            self.audio_feature = self.audio_feature[np.newaxis, :]
        d = os.path.join(self.audio_db_path, user_name)
        os.makedirs(d, exist_ok=True)
        n = len(os.listdir(d))
        path = os.path.join(d, f'{n}.wav').replace('\\', '/')
        import wave as _wave
        with _wave.open(path, 'wb') as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(seg.sample_rate)
            w.writeframes((np.clip(seg.samples, -1, 1) * 32767).astype('<i2').tobytes())
        self.users_audio_path.append(path)
        self.users_name.append(user_name)
        self.__write_index()
        self.__refresh_means()
        return True, "注册成功"

    def recognition(self, audio_data, threshold=None, sample_rate=16000):
        """声纹识别 (predict.py:311-333) -> [name-or-None, score-or-None]"""
        if threshold:
            self.threshold = threshold
        feature = self.predict(audio_data, sample_rate=sample_rate)
        return self.__retrieval(np_feature=[feature])[0]

    def get_users(self):
        return self.users_name

    def remove_user(self, user_name):
        """predict.py:343-363"""
        if user_name not in self.users_name:
            return False
        idx = [i for i, n in enumerate(self.users_name) if n == user_name]
        for i in sorted(idx, reverse=True):
            self.users_name.pop(i)
            self.users_audio_path.pop(i)
        self.audio_feature = np.delete(self.audio_feature, idx, axis=0)
        self.__write_index()
        shutil.rmtree(os.path.join(self.audio_db_path, user_name), ignore_errors=True)
        self.__refresh_means()
        return True

    def speaker_diarization(self, audio_data, sample_rate=16000, speaker_num=None, search_audio_db=False):
        """说话人日志识别 (predict.py:365-395) -> [{'speaker': id or name, 'start': s, 'end': s}, ...]"""
        input_data = self._condition_host(self._load_audio(audio_data=audio_data, sample_rate=sample_rate))
        # the 16 kHz chunks go to predict_batch with the caller's sample_rate, as in the reference (predict.py:379): a
        # caller at another rate has them resampled a second time
        segments = self.speaker_diarize.segments_audio(input_data)
        features = self.predict_batch([seg[2] for seg in segments], sample_rate=sample_rate)
        labels, spk_center_embeddings = self.speaker_diarize.clustering(features, speaker_num=speaker_num)
        outputs = self.speaker_diarize.postprocess(segments, labels)
        if search_audio_db:
            assert self.audio_feature is not None, "数据库中没有音频数据，请先指定说话人特征数据库或者注册说话人"
            names = self.__retrieval(np_feature=spk_center_embeddings)
            outputs = [{'speaker': names[o['speaker']][0] if names[o['speaker']][0] else f"陌生人{o['speaker']}",
                        'start': o['start'], 'end': o['end']} for o in outputs]
        return outputs
