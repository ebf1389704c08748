"""MVectorTrainer -- the two hot-path callers: ``extract_features`` (reference: mvector/trainer.py:146-175) and
``evaluate`` (trainer.py:403-485).

``extract_features`` walks the train / enroll / trials lists (``path\\tlabel`` lines), runs the front-end on every file
exactly like ``MVectorDataset.__getitem__`` does in ``mode='extract_feature'`` (reader.py:82-107: skip files shorter than
``min_duration``, resample, dB-normalise, crop to ``max_duration`` from the start, featurize ONE utterance -> [T, F]) and
writes the reference's feature cache: ``<save_dir>/<label>/<ms timestamp>.npy`` float32 [T, F] plus a
``*_features.txt`` list that the reference's reader consumes (reader.py:76-81).  The front-end runs on the fused sm_90a
kernel.

``evaluate`` embeds the enroll and trials lists and scores every trial against every enrolment.  Data semantics follow
``MVectorDataset(mode='eval')`` + ``collate_fn`` (reader.py:63-109,127-144; collate_fn.py:5-24): lists are sorted by
duration (``np.argsort``), every file is featurized ALONE (CMN over its own frames, no mask), cropped from the start to
``eval_conf.max_duration``, then ``eval_conf.batch_size`` consecutive features are zero-padded at the FEATURE level to
the longest in the batch and fed to the backbone -- padded frames do reach the pooling layer, exactly as in the
reference.  Front-end, backbone and cosine scores run on the sm_90a kernels.  EER / minDCF (trainer.py:462-468,
metric/metrics.py) run on the device too once the score matrix has ``DEVICE_METRICS_MIN`` entries (csrc/verify.cu: a
stable radix sort of the scores and exact fp64 curves; no score copy, no host label matrix); smaller matrices take the
numpy glue.  Training and export are outside the embedding-extraction path and raise."""
import os
import time

import numpy as np
import torch
import yaml
from loguru import logger

from .audio import AudioSegment, EncodedSegment, FlacSegment, check_status, device_samples
from .data_utils.featurizer import AudioFeaturizer
from .metric.metrics import compute_dcf, compute_eer, compute_fnr_fpr
from .utils.utils import dict_to_object, print_arguments


def plan_groups(sizes, bs, max_files, max_floats):
    """[lo, hi) ranges over len(sizes) items in order, each run through the device as one group: a whole number of
    ``bs``-item slices (the last group may end short), at most ``max_files`` items (rounded down to a multiple of bs, one
    slice at least) and, once it holds a slice, no slice that would take its padded rectangle -- items times the
    largest of their ``sizes``, the floats of every buffer a group pads to its widest row -- past ``max_floats``.  So
    one long item never widens the rows of many short ones: it ends the group before it and starts a narrow one."""
    n = len(sizes)
    cap = max(bs, max_files // bs * bs)
    groups, lo = [], 0
    while lo < n:
        hi, width = lo, 0
        while hi < n and hi - lo < cap:
            nxt = min(hi + bs, n)
            w = max(width, max(sizes[hi:nxt]))
            if hi > lo and (nxt - lo) * w > max_floats:
                break
            hi, width = nxt, w
        groups.append((lo, hi))
        lo = hi
    return groups


def resolve_sources(n, usable):
    """reader.py:86-88,102-106: list index i is served by the first entry j = i, i + 1, ... (wrapping) with ``usable(j)``
    -> [j for every i], or None for every index when no entry is usable.  ``usable`` is asked once per entry."""
    ok = {}

    def good(j):
        if j not in ok:
            ok[j] = usable(j)
        return ok[j]

    out = [None] * n
    nxt = None                      # the source of index i + 1, walking down from the end
    for i in range(n - 1, -1, -1):
        if good(i):
            nxt = i
        out[i] = nxt
    if nxt is None:
        return out
    for i in range(n - 1, -1, -1):  # indices past the last usable entry wrap to the first usable one
        if out[i] is not None:
            break
        out[i] = nxt
    return out


def _eval_sorted(data_list):
    """sort_list (reader.py:127-144): the list's (path, label) entries sorted by duration (frames for .npy features),
    those lengths and the files' native rates (0 for .npy), from the headers alone."""
    with open(data_list, 'r', encoding='utf-8') as f:
        lines = f.readlines()
    entries, lengths, rates = [], [], []
    for line in lines:
        path, label = line.replace('\n', '').split('\t')
        if path.endswith('.npy'):
            lengths.append(np.load(path, mmap_mode='r').shape[0])
            rates.append(0)
        else:
            seg = AudioSegment.from_file(path)
            lengths.append(seg.duration)
            rates.append(seg.sample_rate)
        entries.append((path, int(label)))
    order = np.argsort(lengths)
    return [entries[i] for i in order], [lengths[i] for i in order], [rates[i] for i in order]


class MVectorTrainer(object):
    # score-matrix size (n_trials * n_enroll) from which evaluate computes EER / minDCF on the device (DESIGN.md 8.2)
    DEVICE_METRICS_MIN = 1 << 20
    # evaluate / extract_features run the device path on groups of files: decode, conditioning and front-end once per
    # group.  At most MAX_GROUP files, and at most MAX_GROUP_FLOATS (128 MB) in each buffer the group pads to its widest
    # row (plan_groups, _row_floats).
    MAX_GROUP = 256
    MAX_GROUP_FLOATS = 1 << 25

    def __init__(self, configs, use_gpu=True, data_augment_configs=None):
        if use_gpu:
            assert torch.cuda.is_available(), 'GPU不可用'
        else:
            raise RuntimeError('use_gpu=False: the GPU-native path has no CPU implementation')
        if isinstance(configs, str):
            with open(configs, 'r', encoding='utf-8') as f:
                configs = yaml.load(f.read(), Loader=yaml.FullLoader)
            print_arguments(configs=configs)
        self.configs = dict_to_object(configs)
        self.use_gpu = use_gpu
        self.audio_featurizer = None
        self.model = None
        self.stop_eval = False

    def extract_features(self, save_dir='dataset/features', max_duration=100):
        """提取特征保存文件 (trainer.py:146-175)"""
        pc = self.configs.preprocess_conf
        self.audio_featurizer = AudioFeaturizer(feature_method=pc.feature_method,
                                                use_hf_model=pc.get('use_hf_model', False),
                                                method_args=pc.get('method_args', {}))
        ds = self.configs.dataset_conf.get('dataset', {})
        min_duration = ds.get('min_duration', 0.5)
        sample_rate = ds.get('sample_rate', 16000)
        use_db, target_db = ds.get('use_dB_normalization', True), ds.get('target_dB', -20)
        eng = self.audio_featurizer.engine
        for data_list in (self.configs.dataset_conf.train_list, self.configs.dataset_conf.enroll_list,
                          self.configs.dataset_conf.trials_list):
            with open(data_list, 'r', encoding='utf-8') as f:
                lines = [ln for ln in f.read().splitlines() if ln.strip()]
            paths = [ln.split('\t')[0] for ln in lines]
            labels = [int(ln.split('\t')[1]) for ln in lines]

            dur, rate = {}, {}

            def usable(j):
                try:
                    seg = AudioSegment.from_file(paths[j])
                    dur[j], rate[j] = seg.duration, seg.sample_rate
                    return dur[j] >= min_duration
                except Exception as e:  # noqa: BLE001  (the reference logs and moves on, reader.py:103-106)
                    logger.error(f"[{paths[j]}]特征提取失败，错误信息：{e}")
                    return False

            src = resolve_sources(len(lines), usable)         # header durations only: nothing is decoded here
            if src and src[0] is None:
                raise RuntimeError('no usable audio file in ' + data_list)
            save_data_list = data_list.replace('.txt', '_features.txt')
            with open(save_data_list, 'w', encoding='utf-8') as out:
                for lo, hi in plan_groups([self._row_floats(dur[j], rate[j], sample_rate, max_duration) for j in src], 1,
                                          self.MAX_GROUP, self.MAX_GROUP_FLOATS):
                    while True:
                        segs = [AudioSegment.from_file(paths[src[i]]) for i in range(lo, hi)]
                        try:
                            feats, tb, row = self._group_features(segs, sample_rate, target_db if use_db else None,
                                                             max_duration, eng)
                            break
                        except _Refused as r:
                            # a file the device decode refuses: its indices take the per-file rule, which decodes the
                            # candidates one at a time and so skips the refused file
                            for k in r.rows:
                                i, bad = lo + k, src[lo + k]
                                j = self._resolve_decoding(paths, min_duration, i, eng)
                                if j == bad:
                                    raise
                                src[i] = j
                    host = feats.cpu().numpy()                  # one device-to-host copy per group
                    for k, i in enumerate(range(lo, hi)):
                        label = labels[src[i]]
                        stamp = int(time.time() * 1000)
                        save_path = os.path.join(save_dir, str(label), f'{stamp}.npy').replace('\\', '/')
                        while os.path.exists(save_path):      # the reference's ms timestamp collides at GPU speed
                            stamp += 1
                            save_path = os.path.join(save_dir, str(label), f'{stamp}.npy').replace('\\', '/')
                        os.makedirs(os.path.dirname(save_path), exist_ok=True)
                        np.save(save_path, host[row[k], :tb[row[k]]])
                        out.write(f'{save_path}\t{label}\n')
            logger.info(f'{data_list}列表中的数据已提取特征完成，新列表为：{save_data_list}')

    @staticmethod
    def _resolve_decoding(paths, min_duration, idx, eng):
        """reader.py:86-88,102-106 for list index ``idx``, a FLAC candidate decoded on the device first so that a corrupt
        one is skipped like a bad WAV -> the index of the entry that serves it."""
        j = idx
        for _ in range(len(paths)):
            try:
                cand = AudioSegment.from_file(paths[j])
                if cand.duration >= min_duration:
                    if isinstance(cand, FlacSegment):
                        cand.decode_device(eng)
                    return j
            except Exception as e:  # noqa: BLE001  (the reference logs and moves on, reader.py:103-106)
                logger.error(f"[{paths[j]}]特征提取失败，错误信息：{e}")
            j = j + 1 if j < len(paths) - 1 else 0
        raise RuntimeError('no usable audio file')

    def train(self, *args, **kwargs):
        raise NotImplementedError('training is outside the GPU embedding-extraction path (SURVEY.md section 2, row 7)')

    # ------------------------------------------------------------------ evaluate (trainer.py:403-485)
    def _setup_eval(self):
        from .engine import Engine
        from .models import build_model
        pc = self.configs.preprocess_conf
        self._engine = Engine(torch.cuda.current_device())
        self._device = self._engine.device
        self.audio_featurizer = AudioFeaturizer(feature_method=pc.feature_method,
                                                use_hf_model=pc.get('use_hf_model', False),
                                                method_args=pc.get('method_args', {}), engine=self._engine)
        self.model = build_model(input_size=self.audio_featurizer.feature_dim, configs=self.configs)
        self.model.engine = self._engine

    def _eval_order(self, data_list):
        """Reference eval order (sort_list, reader.py:127-144): entries sorted by duration (frames for .npy features).  Only
        (path, label) is kept -- audio is decoded again, one group at a time, when it is embedded."""
        return _eval_sorted(data_list)[0]

    def _eval_feature(self, path):
        """One item's feature [T, F] on the device (reader.py:76-100, eval mode)."""
        ds = self.configs.dataset_conf.get('dataset', {})
        sample_rate = ds.get('sample_rate', 16000)
        use_db, target_db = ds.get('use_dB_normalization', True), ds.get('target_dB', -20)
        max_duration = self.configs.dataset_conf.eval_conf.max_duration          # trainer.py:126
        if path.endswith('.npy'):                                                # reader.py:76-81
            # get_crop_feature_len (reader.py:119-124): frames of a max_duration-long waveform
            max_feature_len = self.audio_featurizer.num_frames(int(max_duration * sample_rate))
            return torch.from_numpy(np.asarray(np.load(path)[:max_feature_len], dtype=np.float32)).to(self._device)
        seg = AudioSegment.from_file(path)
        return self.audio_featurizer(self._condition(seg, sample_rate, target_db if use_db else None, max_duration,
                                                     getattr(self, '_engine', None))).squeeze(0)

    @staticmethod
    def _condition(seg, sample_rate, target_db, max_duration, eng):
        """reader.py:82-107 for one decoded file: resample the WHOLE file to ``sample_rate`` and dB-normalise it
        (``target_db`` not None) on the device of ``eng``, then crop it to ``max_duration`` from the start -> [n] device
        float32 (Engine.condition; a file already at the rate with normalisation off is uploaded as it is).
        ``eng`` None is a trainer without a device engine -- the host-logic tests drive evaluate with CPU oracle
        stand-ins for the featurizer and backbone -- which conditions with AudioSegment on the host (CPU tensor)."""
        if eng is None:
            if seg.sample_rate != sample_rate:
                seg.resample(sample_rate)
            if target_db is not None:
                seg.normalize(target_db=target_db)
            n = seg.samples.shape[0]
            crop = int(max_duration * sample_rate) if n / float(sample_rate) > max_duration else n
            return torch.from_numpy(seg.samples[:crop])
        x = device_samples(seg, eng)                           # a FLAC file is decoded on the device
        n = x.shape[0]
        if seg.sample_rate != sample_rate or target_db is not None:
            y, n_out, flags = eng.condition(x.unsqueeze(0), [n], [seg.sample_rate], sample_rate, target_db)
            if flags is not None and int(flags.cpu()[0]):
                seg.resample(sample_rate)
                seg.normalize(target_db=target_db)            # raises AudioSegment.normalize's ValueError
            n = int(n_out[0])
            x = y[0]
        if n / float(sample_rate) > max_duration:             # crop(mode='eval'): from the start
            n = int(max_duration * sample_rate)
        return x[:n]

    def _row_floats(self, duration, rate, sample_rate, max_duration):
        """Floats one file of ``duration`` s at ``rate`` Hz takes in each buffer _group_features pads to the group's
        widest row: its native row (uncropped), its conditioned row (uncropped) and its features, or the MFCC mel values
        of the front-end's scratch."""
        fz = self.audio_featurizer
        frames = fz.num_frames(int(min(duration, max_duration) * sample_rate))
        return int(max(duration * rate, duration * sample_rate, frames * max(fz.feature_dim, fz.feat_fun.n_mels))) + 1

    def _group_features(self, segs, sample_rate, target_db, max_duration, eng):
        """reader.py:82-107 for a group of files at once -> (features CUDA [n, T, F], each row one file featurized alone
        and +0.0 past its T_b frames; T_b numpy [n] by row; row numpy [n]: file i is feature row row[i]).  Each codec class is decoded in one device decode, files read by the
        ``wave`` reader are uploaded, one Engine.condition resamples (each row from its own rate) and dB-normalises
        them, each row is cropped to max_duration from the start, and one forward_each featurizes them.  A refused
        decode raises _Refused, check_status's ValueError naming the files; a row the gain flags raises
        AudioSegment.normalize's ValueError, as _condition does."""
        n = len(segs)
        enc = [isinstance(s, EncodedSegment) and s._samples is None for s in segs]
        classes = {}
        for i, s in enumerate(segs):
            classes.setdefault(s.batch_type if enc[i] else None, []).append(i)
        order = [i for rows in classes.values() for i in rows]          # device row k holds file order[k]
        n_in = np.zeros(n, dtype=np.int64)
        batches = {}
        for bt, rows in classes.items():
            if bt is not None:
                batches[bt] = bt([segs[i].data for i in rows], [segs[i].info for i in rows], eng.device,
                                 [segs[i].name for i in rows])
                n_in[rows] = batches[bt].lengths
            else:
                n_in[rows] = [segs[i].samples.shape[0] for i in rows]
        ld = max(int(n_in.max()), 1)
        x = torch.empty(n, ld, dtype=torch.float32, device=eng.device)
        status = torch.zeros(n, dtype=torch.int32, device=eng.device)
        k = 0
        for bt, rows in classes.items():
            if bt is not None:
                batches[bt].decode_into(eng, x[k:k + len(rows)], ld, status[k:k + len(rows)])
            else:
                host = np.zeros((len(rows), ld), dtype=np.float32)
                for r, i in enumerate(rows):
                    host[r, :n_in[i]] = segs[i].samples
                x[k:k + len(rows)].copy_(torch.from_numpy(host))
            k += len(rows)
        if batches:
            st = status.cpu().numpy()
            if st.any():
                names = [segs[i].name if enc[i] else '' for i in order]
                bad = [order[r] for r in np.flatnonzero(st)]
                try:
                    check_status(st, names, '/'.join(b.label for b in batches.values()), 'file')
                except ValueError as err:
                    raise _Refused(bad, str(err)) from None
        rates = np.array([segs[i].sample_rate for i in order], dtype=np.int64)
        lens = n_in[order]
        if (rates != sample_rate).any() or target_db is not None:
            x, lens, flags = eng.condition(x, lens, rates, sample_rate, target_db)
            if flags is not None:
                bad = np.flatnonzero(flags.cpu().numpy())
                if bad.size:
                    seg = segs[order[int(bad[0])]]
                    seg.resample(sample_rate)
                    seg.normalize(target_db=target_db)             # raises AudioSegment.normalize's ValueError
                    raise ValueError(f'cannot normalise to {target_db} dB: the gain of row {int(bad[0])} exceeds 300 dB')
        crop = int(max_duration * sample_rate)
        lens = np.where(lens / float(sample_rate) > max_duration, crop, lens)   # crop(mode='eval'): from the start
        feats, tb = self.audio_featurizer.forward_each(x, lens)
        row = np.empty(n, dtype=np.int64)
        row[order] = np.arange(n)
        return feats, tb, row

    def _embed_list(self, data_list):
        """Embeddings of one list in eval order, one eval_conf.batch_size batch at a time: decode -> featurize singly ->
        zero-pad the FEATURES to the batch's longest item (collate_fn.py:12-19) -> backbone.  With a device engine the
        files run in groups of whole batches (_group_features); a trainer without one (CPU stand-ins) featurizes file by
        file.  The padding is device-to-device copies (no library kernel on the path)."""
        if getattr(self, '_engine', None) is None:
            return self._embed_list_each(data_list)
        entries, lengths, rates = _eval_sorted(data_list)
        ds = self.configs.dataset_conf.get('dataset', {})
        sample_rate = ds.get('sample_rate', 16000)
        use_db, target_db = ds.get('use_dB_normalization', True), ds.get('target_dB', -20)
        max_duration = self.configs.dataset_conf.eval_conf.max_duration
        bs = self.configs.dataset_conf.eval_conf.batch_size
        sizes = [0 if p.endswith('.npy') else self._row_floats(d, r, sample_rate, max_duration)
                 for (p, _), d, r in zip(entries, lengths, rates)]
        feats, labels = [], []
        for lo, hi in plan_groups(sizes, bs, self.MAX_GROUP, self.MAX_GROUP_FLOATS):
            if self.stop_eval:
                break
            audio = [i for i in range(lo, hi) if not entries[i][0].endswith('.npy')]
            row = {}
            if audio:
                gf, tb, frow = self._group_features([AudioSegment.from_file(entries[i][0]) for i in audio], sample_rate,
                                              target_db if use_db else None, max_duration, self._engine)
                row = {i: int(frow[k]) for k, i in enumerate(audio)}
            for s in range(lo, min(hi, len(entries)), bs):
                if self.stop_eval:
                    break
                idx = list(range(s, min(s + bs, hi)))
                if all(i in row for i in idx):
                    # rows are +0.0 past their own frames already: each is one contiguous copy of its first tmax frames
                    tmax = int(max(tb[row[i]] for i in idx))
                    x = torch.empty((len(idx), tmax, gf.shape[2]), dtype=torch.float32, device=self._device)
                    for k, i in enumerate(idx):
                        x[k].copy_(gf[row[i], :tmax])
                else:
                    x = self._zero_pad_features([gf[row[i], :tb[row[i]]] if i in row else self._eval_feature(entries[i][0])
                                                 for i in idx])
                feats.append(self.model(x).cpu().numpy())
                labels.extend(entries[i][1] for i in idx)
        return np.concatenate(feats), np.asarray(labels, dtype=np.int32)

    def _embed_list_each(self, data_list):
        """_embed_list file by file: decode -> featurize singly -> zero-pad -> backbone, one batch at a time."""
        entries = self._eval_order(data_list)
        bs = self.configs.dataset_conf.eval_conf.batch_size
        feats, labels = [], []
        for s in range(0, len(entries), bs):
            if self.stop_eval:
                break
            chunk = [(self._eval_feature(path), label) for path, label in entries[s:s + bs]]
            feats.append(self.model(self._zero_pad_features([f for f, _ in chunk])).cpu().numpy())
            labels.extend(lb for _, lb in chunk)
        return np.concatenate(feats), np.asarray(labels, dtype=np.int32)

    def _zero_pad_features(self, items):
        """collate_fn.py:12-19 on the device: [T_i, F] features -> zero-padded [B, Tmax, F] (memset + D2D row copies)."""
        import ctypes as C
        from . import _lib as L
        tmax = max(f.shape[0] for f in items)
        x = torch.empty((len(items), tmax, items[0].shape[1]), dtype=torch.float32, device=self._device)
        rc = L.lib().vp_device_zero(C.c_void_p(x.data_ptr()), x.numel() * 4, self._engine.stream_ptr())
        if rc != L.VP_OK:
            raise L.VpError(rc, 'vp_device_zero failed')
        for i, f in enumerate(items):
            x[i, :f.shape[0]].copy_(f)                                           # contiguous rows: a D2D memcpy
        return x

    def _cosine_scores(self, trials, enroll):
        """trainer.py:454-461 (sklearn cosine_similarity of every trial against every enrolment) on the device."""
        return self._engine.cosine_scores(trials, enroll).cpu().numpy()

    def evaluate(self, resume_model=None, save_image_path=None):
        """评估模型 (trainer.py:403-485) -> (eer, min_dcf, threshold)"""
        from .utils.checkpoint import load_pretrained
        if self.model is None:
            self._setup_eval()
        if resume_model is not None:
            if os.path.isdir(resume_model):
                resume_model = os.path.join(resume_model, 'model.pth')
            assert os.path.exists(resume_model), f"{resume_model} 模型不存在！"
            self.model = load_pretrained(self.model, resume_model, use_gpu=self.use_gpu)
        self.model.eval()
        enroll_features, enroll_labels = self._embed_list(self.configs.dataset_conf.enroll_list)
        trials_features, trials_labels = self._embed_list(self.configs.dataset_conf.trials_list)
        if self.stop_eval:
            return -1, -1, -1
        logger.info('开始对比音频特征...')
        # cosine_similarity of every trial against every enrolment (trainer.py:454-461), trial-major order, on the device
        if len(trials_labels) * len(enroll_labels) >= self.DEVICE_METRICS_MIN:
            scores = self._engine.cosine_scores(trials_features, enroll_features)
            out = self._engine.verification_metrics(scores.reshape(-1), trial_labels=trials_labels,
                                                    enroll_labels=enroll_labels, curves=bool(save_image_path))
            eer, min_dcf, threshold = out[:3]
            if save_image_path:
                fnr, fpr, thresholds = out[3:]
        else:
            all_score = self._cosine_scores(trials_features, enroll_features).reshape(-1)
            all_labels = (trials_labels[:, None] == enroll_labels[None, :]).astype(np.int32).reshape(-1)
            fnr, fpr, thresholds = compute_fnr_fpr(all_score, all_labels)
            eer, threshold = compute_eer(fnr, fpr, all_score)
            min_dcf = compute_dcf(fnr, fpr)
        eer, min_dcf, threshold = float(eer), float(min_dcf), float(threshold)
        if save_image_path:                                                       # trainer.py:471-484
            import matplotlib.pyplot as plt
            at = int(np.flatnonzero(np.asarray(thresholds) == threshold)[0])
            plt.plot(thresholds, fnr, color='blue', linestyle='-', label='fnr')
            plt.plot(thresholds, fpr, color='red', linestyle='-', label='fpr')
            plt.plot(threshold, fpr[at], 'ro-')
            plt.text(threshold, fpr[at], (round(threshold, 3), round(fpr[at], 5)), color='red')
            plt.xlabel('threshold')
            plt.title('fnr and fpr')
            plt.grid(True)
            os.makedirs(save_image_path, exist_ok=True)
            plt.savefig(os.path.join(save_image_path, 'result.png'))
            logger.info(f"结果图以保存在：{os.path.join(save_image_path, 'result.png')}")
        return eer, min_dcf, threshold

    def export(self, *args, **kwargs):
        raise NotImplementedError('torch.jit export does not apply to the C-ABI path')


class _Refused(ValueError):
    """check_status's ValueError for a group whose device decode refused ``rows`` (indices into the group)."""

    def __init__(self, rows, msg):
        super().__init__(msg)
        self.rows = rows
