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

from .audio import AudioSegment
from .data_utils.featurizer import AudioFeaturizer
from .metric.metrics import compute_dcf, compute_eer, compute_fnr_fpr
from .utils.utils import dict_to_object, print_arguments


class MVectorTrainer(object):
    # score-matrix size (n_trials * n_enroll) from which evaluate computes EER / minDCF on the device (DESIGN.md 8.2)
    DEVICE_METRICS_MIN = 1 << 20

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
        for data_list in (self.configs.dataset_conf.train_list, self.configs.dataset_conf.enroll_list,
                          self.configs.dataset_conf.trials_list):
            with open(data_list, 'r', encoding='utf-8') as f:
                lines = [ln for ln in f.read().splitlines() if ln.strip()]
            save_data_list = data_list.replace('.txt', '_features.txt')
            with open(save_data_list, 'w', encoding='utf-8') as out:
                for idx in range(len(lines)):
                    # reader.py:86-88,102-106: a short / unreadable file is replaced by its successor in the list
                    j, seg = idx, None
                    for _ in range(len(lines)):
                        path, label = lines[j].split('\t')
                        try:
                            cand = AudioSegment.from_file(path)
                            if cand.duration >= min_duration:
                                seg = cand
                                break
                        except Exception as e:  # noqa: BLE001  (the reference logs and moves on, reader.py:103-106)
                            logger.error(f"[{path}]特征提取失败，错误信息：{e}")
                        j = j + 1 if j < len(lines) - 1 else 0
                    if seg is None:
                        raise RuntimeError('no usable audio file in ' + data_list)
                    wave = self._condition(seg, sample_rate, target_db if use_db else None, max_duration,
                                           self.audio_featurizer.engine)
                    feature = self.audio_featurizer(wave).squeeze(0).cpu().numpy()
                    label = int(label)
                    stamp = int(time.time() * 1000)
                    save_path = os.path.join(save_dir, str(label), f'{stamp}.npy').replace('\\', '/')
                    while os.path.exists(save_path):      # the reference's ms timestamp collides at GPU speed
                        stamp += 1
                        save_path = os.path.join(save_dir, str(label), f'{stamp}.npy').replace('\\', '/')
                    os.makedirs(os.path.dirname(save_path), exist_ok=True)
                    np.save(save_path, feature.astype(np.float32))
                    out.write(f'{save_path}\t{label}\n')
            logger.info(f'{data_list}列表中的数据已提取特征完成，新列表为：{save_data_list}')

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
        (path, label, length) is kept -- audio is decoded again, one batch at a time, when it is embedded."""
        with open(data_list, 'r', encoding='utf-8') as f:
            lines = f.readlines()
        entries, lengths = [], []
        for line in lines:
            path, label = line.replace('\n', '').split('\t')
            if path.endswith('.npy'):
                lengths.append(np.load(path, mmap_mode='r').shape[0])
            else:
                lengths.append(AudioSegment.from_file(path).duration)
            entries.append((path, int(label)))
        return [entries[i] for i in np.argsort(lengths)]

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
        x = torch.from_numpy(np.ascontiguousarray(seg.samples, dtype=np.float32)).to(eng.device)
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

    def _embed_list(self, data_list):
        """Embeddings of one list in eval order, one eval_conf.batch_size batch at a time: decode -> featurize singly ->
        zero-pad the FEATURES to the batch's longest item (collate_fn.py:12-19) -> backbone.  Host and device memory stay
        O(batch); the padding is a memset + device-to-device copies (no library kernel on the path)."""
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
