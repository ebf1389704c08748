"""Speaker-diarization glue around predict_batch (reference: mvector/infer_utils/speaker_diarization.py:9-310, itself
adapted from ModelScope).  The heavy step -- one embedding per 1.5 s chunk -- is ``MVectorPredictor.predict_batch`` on the
sm_90a path; everything here is small host-side numpy / scipy / sklearn work on [n_chunks, embd] arrays, restated with
the same interfaces, defaults and results as the reference classes:

  SpeakerDiarization.segments_audio   VAD segments -> 1.5 s chunks every 0.75 s, last chunk right-aligned (:24-89)
  SpeakerDiarization.clustering       spectral clustering -> relabel by first appearance -> speaker centres -> merge centres
                                      whose cosine exceeds merge_threshold (:91-135)
  SpeakerDiarization.postprocess      merge consecutive chunks of one speaker, split overlaps at the midpoint, absorb
                                      segments shorter than 1 s into a neighbour (:137-214)
  SpectralCluster                     cosine affinity -> keep the top p-fraction per row -> symmetrise -> unnormalised
                                      Laplacian -> eigengap (or oracle) speaker count -> k-means on the spectral
                                      embedding (:217-310); MVectorPredictor runs everything up to the eigenvectors on
                                      the device (csrc/spectral.cu, Engine.spectral_embedding)

``AudioSegment.vad`` (yeaudio's model-based VAD) is outside the parity boundary (SURVEY.md 8c); mvector.audio provides an
energy-based stand-in with the same return format."""
import numpy as np
import scipy.linalg
from sklearn.cluster import k_means


class SpectralCluster:
    def __init__(self, min_num_spks=1, max_num_spks=15, pval=0.022):
        self.min_num_spks = min_num_spks
        self.max_num_spks = max_num_spks
        self.pval = pval

    # Optional device implementation of the whole spectral stage (MVectorPredictor installs Engine.spectral_embedding):
    #   spectral_fn(X [n, D] float32, n_drop, n_eig, k_fn) -> (the n_eig smallest Laplacian eigenvalues, their first
    #   k = k_fn(eigenvalues) eigenvectors [n, k]).  None: everything below runs on the host, as in the reference.
    spectral_fn = None

    def __call__(self, X, oracle_num=None):
        if self.spectral_fn is not None:
            n = len(X)
            _, emb = self.spectral_fn(np.asarray(X, dtype=np.float32), self.n_drop(n), min(n, self.max_num_spks + 1),
                                      lambda lambdas: self.num_speakers(lambdas, oracle_num))
            # float32, the dtype the host path's (and the reference's) eigenvectors have: same k-means++ draws
            return self.cluster_embs(np.asarray(emb, dtype=np.float32), emb.shape[1])
        sim = self.get_sim_mat(X)
        affinity = self.p_pruning(sim)
        affinity = 0.5 * (affinity + affinity.T)
        emb, k = self.get_spec_embs(self.get_laplacian(affinity), oracle_num)
        return self.cluster_embs(emb, k)

    @staticmethod
    def get_sim_mat(X):
        """Cosine similarity of every pair of rows (sklearn cosine_similarity: normalise, then one matmul)."""
        X = np.asarray(X)
        n = np.linalg.norm(X, axis=1, keepdims=True)
        Xn = X / np.where(n == 0, 1, n)
        return Xn @ Xn.T

    def n_drop(self, n):
        """Entries p_pruning zeroes per row, as Python evaluates the reference's slice (a negative bound counts from
        the end: n = 4 drops 2)."""
        pval = 6.0 / n if n * self.pval < 6 else self.pval
        return len(range(n)[:int((1 - pval) * n)])

    def p_pruning(self, A):
        """Zero all but the largest ceil-ish p-fraction of every row (at least 6 entries survive)."""
        n = A.shape[0]
        pval = 6.0 / n if n * self.pval < 6 else self.pval
        n_drop = int((1 - pval) * n)
        drop = np.argsort(A, axis=1)[:, :n_drop]
        np.put_along_axis(A, drop, 0, axis=1)
        return A

    @staticmethod
    def get_laplacian(M):
        np.fill_diagonal(M, 0)
        return np.diag(np.abs(M).sum(axis=1)) - M

    def get_spec_embs(self, L, k_oracle=None):
        lambdas, vecs = scipy.linalg.eigh(L)
        k = self.num_speakers(lambdas, k_oracle)
        return vecs[:, :k], k

    def num_speakers(self, lambdas, k_oracle=None):
        """k_oracle, or the position of the largest gap among eigenvalues min_num_spks .. max_num_spks + 1."""
        if k_oracle is not None:
            return k_oracle
        gaps = self.get_eigen_gaps(lambdas[self.min_num_spks - 1:self.max_num_spks + 1])
        return int(np.argmax(gaps)) + self.min_num_spks

    @staticmethod
    def cluster_embs(emb, k):
        return k_means(emb, k, n_init='auto')[1]

    @staticmethod
    def get_eigen_gaps(eig_vals):
        v = [float(x) for x in eig_vals]
        return [b - a for a, b in zip(v[:-1], v[1:])]


class SpeakerDiarization(object):
    def __init__(self, seg_duration=1.5, seg_shift=0.75, sample_rate=16000, merge_threshold=0.78):
        self.seg_duration = seg_duration
        self.seg_shift = seg_shift
        self.sample_rate = sample_rate
        self.merge_threshold = merge_threshold
        self.spectral_cluster = SpectralCluster()

    def set_spectral(self, spectral_fn):
        """Install a device implementation of the clustering's spectral stage (SpectralCluster.spectral_fn; None: the
        host path)."""
        self.spectral_cluster.spectral_fn = spectral_fn

    # ------------------------------------------------------------------ segmentation
    def segments_audio(self, audio_segment):
        """-> [[start s, end s, samples of one chunk], ...] over the voiced parts of the recording."""
        samples = audio_segment.samples
        self.sample_rate = sr = audio_segment.sample_rate
        voiced = []
        for t in audio_segment.vad(return_seconds=True):
            st, ed = round(t['start'], 3), round(t['end'], 3)
            voiced.append([st, ed, samples[int(st * sr):int(ed * sr)]])
        self._check_audio_list(voiced)
        return self._chunk(voiced)

    def _check_audio_list(self, audio):
        total = 0
        for i, (st, ed, data) in enumerate(audio):
            assert ed >= st, '分割的时间戳错误'
            assert isinstance(data, np.ndarray), '数据的类型不正确'
            assert int(ed * self.sample_rate) - int(st * self.sample_rate) == data.shape[0], '时间长度和数据长度不匹配'
            if i > 0:
                assert st >= audio[i - 1][1], 'modelscope error: Wrong time stamps.'
            total += ed - st
        assert total > 5, f'音频时间过段，应当大于5秒，当前长度是{total}秒'

    def _chunk(self, vad_segments):
        size = int(self.seg_duration * self.sample_rate)
        hop = int(self.seg_shift * self.sample_rate)
        out = []
        for seg_st, _, data in vad_segments:
            n = data.shape[0]
            prev_end = 0
            for lo in range(0, n, hop):
                hi = min(lo + size, n)
                if hi <= prev_end:
                    break
                prev_end = hi
                lo = max(0, hi - size)                         # the last chunk is right-aligned to the segment end
                piece = data[lo:hi]
                if piece.shape[0] < size:                      # segment shorter than one chunk: zero-pad
                    piece = np.pad(piece, (0, size - piece.shape[0]), 'constant')
                out.append([lo / self.sample_rate + seg_st, hi / self.sample_rate + seg_st, piece])
        return out

    # ------------------------------------------------------------------ clustering
    def clustering(self, embeddings, speaker_num=None):
        labels = self._correct_labels(self.spectral_cluster(embeddings, oracle_num=speaker_num))
        centres = [embeddings[labels == i].mean(0) for i in range(labels.max() + 1)]
        assert len(centres) > 0
        spk_center_embeddings = np.stack(centres, axis=0)
        labels = self._merge_by_cos(labels, centres, self.merge_threshold)
        return labels, spk_center_embeddings

    @staticmethod
    def _merge_by_cos(labels, spk_center_emb, cos_thr):
        """While the two closest of the first ``labels.max()+1`` centres are more similar than cos_thr, fold the higher
        label into the lower one and close the gap in the numbering.  (Like the reference, the centres themselves are
        not recomputed or re-indexed between rounds.)"""
        assert 0 < cos_thr <= 1
        while True:
            k = labels.max() + 1
            if k == 1:
                break
            c = np.stack([spk_center_emb[i] for i in range(k)], axis=0)
            c = c / np.linalg.norm(c, axis=1, keepdims=True)
            aff = np.triu(c @ c.T, 1)
            a, b = np.unravel_index(np.argmax(aff), aff.shape)
            if aff[a, b] < cos_thr:
                break
            labels = np.where(labels == b, a, np.where(labels > b, labels - 1, labels))
        return labels

    @staticmethod
    def _correct_labels(labels):
        """Renumber clusters by order of first appearance."""
        seen = {}
        return np.array([seen.setdefault(int(v), len(seen)) for v in labels])

    # ------------------------------------------------------------------ post-processing
    def postprocess(self, segments, labels):
        assert len(segments) == len(labels)
        res = self._merge_seque([[seg[0], seg[1], lab] for seg, lab in zip(segments, labels)])
        for prev, cur in zip(res[:-1], res[1:]):               # overlapping neighbours meet at the midpoint
            if prev[1] > cur[0] + 1e-4:
                prev[1] = cur[0] = (cur[0] + prev[1]) / 2
        res = self._smooth(res)
        return [dict(speaker=r[2], start=round(r[0], 3), end=round(r[1], 3)) for r in res]

    @staticmethod
    def _merge_seque(distribute_res):
        res = [distribute_res[0]]
        for item in distribute_res[1:]:
            if item[2] != res[-1][2] or item[0] > res[-1][1]:
                res.append(item)
            else:
                res[-1][1] = item[1]
        return res

    def _smooth(self, res, min_duration=1):
        """Segments shorter than min_duration take the label of the nearer neighbour (ties go left)."""
        last = len(res) - 1
        for i, r in enumerate(res):
            r[0], r[1] = round(r[0], 2), round(r[1], 2)
            if r[1] - r[0] < min_duration:
                if i == 0:
                    r[2] = res[i + 1][2]
                elif i == last:
                    r[2] = res[i - 1][2]
                elif r[0] - res[i - 1][1] <= res[i + 1][0] - r[1]:
                    r[2] = res[i - 1][2]
                else:
                    r[2] = res[i + 1][2]
        return self._merge_seque(res)
