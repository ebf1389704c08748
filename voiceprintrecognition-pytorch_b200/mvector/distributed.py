"""Multi-GPU sharding of the embedding path (SURVEY.md 8e): utterances are independent, so the batch is split into
contiguous index ranges, one per rank (one process per GPU), weights are replicated, and the only collective on the data
path is one all-gather of the per-rank ``[B/R, embd]`` fp32 outputs so that every rank ends up with all embeddings in the
original order.  Ragged batches keep the reference's single-batch semantics (predict.py:244-258: pad to the longest item
of the WHOLE batch, T and the CMN mean follow that padding): every rank pads ITS shard to the global ``Lmax``, which the
host knows from the lengths alone -- no collective, and no rank ever materialises the other ranks' waveforms.

MFCC is the one front-end with a cross-utterance term (torchaudio clamps to (max over the whole call) - top_db): its
sharded form exchanges that one scalar with an all-reduce(MAX) between the mel stage and the DCT
(``AudioFeaturizer.__call__(..., group=...)``, csrc/frontend.cu), so it too is bit-identical to the single-process call.

torch.distributed (NCCL on GPUs, gloo in the CPU tests) is plumbing only; the compute is ``embed_fn`` / the predictor."""
import numpy as np
import torch
import torch.distributed as dist


def _gpu_numa_node(index):
    """NUMA node of CUDA device `index` from sysfs, or None when the platform does not say."""
    try:
        pr = torch.cuda.get_device_properties(index)
        path = f'/sys/bus/pci/devices/{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0/numa_node'
        with open(path) as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except Exception:
        return None


def _parse_cpulist(text):
    cpus = []
    for part in text.strip().split(','):
        if not part:
            continue
        a, _, b = part.partition('-')
        cpus.extend(range(int(a), int(b or a) + 1))
    return cpus


def bind_rank_to_local_cpus(local_rank, local_world):
    """One process per GPU on one host: give every rank its own slice of the host CPUs -- inside the NUMA node its GPU
    hangs off when sysfs tells -- so that the staging threads of the ranks (host gather into pinned memory, H2D) do not
    migrate across sockets or pile onto the same cores, and pinned buffers are first-touched on the GPU's node.  Returns
    the CPU list it bound to (None when nothing was changed)."""
    import os
    try:
        avail = sorted(os.sched_getaffinity(0))
    except AttributeError:
        return None
    if len(avail) < 2 * max(local_world, 1):
        return None
    if local_world <= 1:
        # single process: stay on the NUMA node of the GPU (pinned staging buffers are first-touched there and the
        # gather threads do not wander to the other socket); nothing to do when the platform does not tell
        node = _gpu_numa_node(local_rank) if torch.cuda.is_available() else None
        if node is None:
            return None
        try:
            with open(f'/sys/devices/system/node/node{node}/cpulist') as f:
                cpus = [c for c in _parse_cpulist(f.read()) if c in set(avail)]
            if len(cpus) >= 2:
                os.sched_setaffinity(0, cpus)
                return cpus
        except Exception:
            pass
        return None
    nodes = [_gpu_numa_node(i) for i in range(local_world)] if torch.cuda.is_available() else [None] * local_world
    mine = nodes[local_rank] if local_rank < len(nodes) else None
    pool, peers = avail, list(range(local_world))
    if mine is not None and all(n is not None for n in nodes):
        try:
            with open(f'/sys/devices/system/node/node{mine}/cpulist') as f:
                node_cpus = [c for c in _parse_cpulist(f.read()) if c in set(avail)]
            same = [r for r in range(local_world) if nodes[r] == mine]
            if len(node_cpus) >= 2 * len(same):
                pool, peers = node_cpus, same
        except Exception:
            pass
    k = peers.index(local_rank)
    per = len(pool) // len(peers)
    cpus = pool[k * per:(k + 1) * per]
    try:
        os.sched_setaffinity(0, cpus)
    except OSError:
        return None
    return cpus


def shard_range(n, rank, world):
    """Contiguous, balanced split: the first ``n % world`` ranks get one extra item."""
    base, extra = divmod(n, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


def device_collectives(group=None):
    """True when the group's backend moves CUDA tensors itself (NCCL); with gloo (CPU tests, or two ranks sharing one GPU)
    the tiny payloads of this path are staged through the host."""
    try:
        return 'nccl' in str(dist.get_backend(group)).lower()
    except Exception:
        return False


def pad_to_global_max(waves, lo=0, hi=None, lmax=None):
    """list of 1-D float32 arrays -> (x [hi-lo, Lmax] zero padded, ratio [hi-lo] = len / Lmax) (predict.py:244-255).
    ``lmax`` defaults to the longest item of the WHOLE list; only rows lo..hi are materialised."""
    hi = len(waves) if hi is None else hi
    if lmax is None:
        lmax = max(w.shape[0] for w in waves)
    x = np.zeros((hi - lo, lmax), dtype=np.float32)
    ratio = np.empty(hi - lo, dtype=np.float32)
    for i in range(lo, hi):
        w = waves[i]
        x[i - lo, :w.shape[0]] = w
        ratio[i - lo] = w.shape[0] / lmax
    return x, ratio


def gather_embeddings(local, n, group=None, out=None):
    """``local``: this rank's ``[hi - lo, D]`` embeddings (device tensor, rows of ``shard_range(n, rank, world)``) ->
    the full ``[n, D]`` tensor in the original order on every rank: ONE all-gather (SURVEY.md 8e).  Equal shards (the
    bench's weak-scaling case) go straight into ``out`` / a fresh tensor; uneven shards are padded to the largest shard
    and compacted afterwards."""
    rank, world = _world(group)
    if world == 1:
        return local[:n]
    if local.is_cuda and not device_collectives(group):
        return gather_embeddings(local.cpu(), n, group).to(local.device)
    D = local.shape[1]
    base, extra = divmod(n, world)
    per = base + (1 if extra else 0)
    if extra == 0:
        full = out if out is not None else torch.empty(n, D, dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(full, local.contiguous(), group=group)
        return full
    slot = torch.zeros(per, D, dtype=local.dtype, device=local.device)
    slot[:local.shape[0]] = local
    gathered = torch.empty(world * per, D, dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(gathered, slot, group=group)
    parts = []
    for r in range(world):
        a, b = shard_range(n, r, world)
        parts.append(gathered[r * per: r * per + (b - a)])
    return torch.cat(parts, dim=0)


def embed_sharded(embed_fn, waves, embd_dim, device, group=None):
    """Every rank passes the same ``waves`` list; rank r embeds its shard with ``embed_fn(x[B_r, Lmax], ratio[B_r]) ->
    tensor [B_r, embd_dim] on `device```; returns the full ``[B, embd_dim]`` tensor on every rank."""
    rank, world = _world(group)
    n = len(waves)
    lmax = max(w.shape[0] for w in waves)
    lo, hi = shard_range(n, rank, world)
    local = torch.zeros(hi - lo, embd_dim, dtype=torch.float32, device=device)
    if hi > lo:
        x, ratio = pad_to_global_max(waves, lo, hi, lmax)
        local = embed_fn(x, ratio)
    return gather_embeddings(local, n, group)


def predict_batch_sharded(predictor, audios_data, sample_rate=16000, group=None, as_numpy=True):
    """``MVectorPredictor.predict_batch`` (predict.py:231-265) over all ranks of ``group``: every rank passes the same
    list, loads / stages / embeds only its contiguous shard -- padded to the longest item of the WHOLE list, with the
    whole list's mask ratios -- and one all-gather returns ``[B, embd_dim]`` (order preserved) on every rank.  The result
    is bit-identical to the single-process ``predict_batch`` of the same list.

    Lmax and the ratios need only the other ranks' lengths after resampling, which follow from their native lengths and
    rates (``resampled_length``): a rank decodes its own shard and conditions it (resample, dB normalisation) on its
    device, and never materialises another rank's waveforms."""
    from .audio import resample_ratio, resampled_length
    rank, world = _world(group)
    n = len(audios_data)
    target_sr = predictor.configs.dataset_conf.dataset.sample_rate
    lo, hi = shard_range(n, rank, world)
    ds = predictor.configs.dataset_conf.dataset
    mine = {}
    rates = np.full(n, int(sample_rate), dtype=np.int64)
    if n > 0 and set(map(type, audios_data)) == {np.ndarray}:
        # Raw arrays at the caller's rate: Lmax needs only the lengths of the other ranks' items -- one C-level pass
        # (a Python loop over the WHOLE list costs ~2 us per item: 4 ms per call for 2048 utterances on 8 ranks, which was
        # the whole end-to-end scaling loss of the 8-GPU runs) -- and this rank's own items are used in place when
        # _load_audio would hand them back unchanged (predict.py:196-204), else decoded like any other input
        lens = np.fromiter(map(len, audios_data), dtype=np.int64, count=n)
        short = int(lens.min())
        assert short / float(sample_rate) >= ds.min_duration, f'音频太短，最小应该为{ds.min_duration}s，当前音频为{short / float(sample_rate)}s'
        for i in range(lo, hi):
            a = audios_data[i]
            if a.dtype == np.float32 and a.ndim == 1 and a.flags.c_contiguous:
                mine[i] = a
            else:
                seg = predictor._load_audio(audio_data=a, sample_rate=sample_rate)
                mine[i] = np.ascontiguousarray(seg.samples, dtype=np.float32)
                lens[i] = mine[i].shape[0]
    else:
        lens = np.empty(n, dtype=np.int64)
        for i, a in enumerate(audios_data):
            if type(a) is np.ndarray and a.ndim == 1 and not (lo <= i < hi):
                assert a.shape[0] / float(sample_rate) >= ds.min_duration, \
                    f'音频太短，最小应该为{ds.min_duration}s，当前音频为{a.shape[0] / float(sample_rate)}s'
                lens[i] = a.shape[0]                # another rank's raw array: only its length matters here
                continue
            seg = predictor._load_audio(audio_data=a, sample_rate=sample_rate)
            lens[i] = seg.samples.shape[0]
            if not isinstance(a, np.ndarray):
                rates[i] = seg.sample_rate         # files, bytes and AudioSegments carry their own rate
            if lo <= i < hi:
                mine[i] = np.ascontiguousarray(seg.samples, dtype=np.float32)
    ratio = {r: resample_ratio(r, target_sr) for r in set(rates.tolist())}
    lmax = int(resampled_length(lens, [ratio[r][0] for r in rates.tolist()], [ratio[r][1] for r in rates.tolist()]).max()) \
        if n else 0
    grp = None
    if world > 1:
        grp = group if group is not None else dist.group.WORLD       # MFCC's call-wide clamp maximum spans the ranks
    own = rates[lo:hi].tolist()
    resample = {'rates': own} if any(r != target_sr for r in own) else {}
    local = predictor._embed_waves([mine[i] for i in range(lo, hi)], lmax, masked=True, to_numpy=False, group=grp,
                                   **resample)
    full = gather_embeddings(local, n, group)
    return full.cpu().numpy() if as_numpy else full
