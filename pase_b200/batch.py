"""On-device batch assembly: a drop-in for the reference's DataLoader over
``LibriSpeechSegTupleWavDataset`` (pase/dataset.py:428-513) or ``AmiSegTupleWavDataset``
(516-681, close-talk utterances paired with distant-microphone channels) with ``MIChunkWav`` /
``SingleChunkWav`` (pase/transforms.py:295-436), ``CachedCompose`` (253-292) and
``DictCollater`` (dataset.py:21-89), for a corpus resident in device (or mapped host) memory.

    wavs = WavPool(data_root, data_cfg, 'train')
    batcher = DeviceBatcher.from_train_opts(workers_cfg, 32000, 160, wavs, stats=stats_pkl,
                                            trans_cache=cache_dir, distortions=dist)
    for indices in BatchSampler(RandomSampler(range(len(wavs))), 32, drop_last=True):
        batch = batcher(indices)          # the collated dict the reference's loader yields
    batcher.reset()                       # once per epoch

The host planner draws, per sample and in the reference's order, from Python ``random``,
``np.random`` and torch's default generator (or an explicit triple), exactly what a
``num_workers=0`` loader draws: the zero-speech coin, the context neighbour, the random
utterance, the chunk windows, the random scales, then the sample's distortions.  It packs the
draws into one int64 table; the device side is one upload and a fixed list of launches
(csrc/batch.cu, the targets and the distortions), so it can be captured in a CUDA graph.

Kept from the reference on purpose: the neighbour lists shrink as utterances are visited
(``neighbors.remove``), the last window start L - T is never drawn, a silent chunk scales to
0/0 = NaN, cached features are sliced ``[beg // hop, (beg + T) // hop)`` and not z-normed.

AMI (``dataset="ami"``): with ``ihm2sdm`` channel keys the pool holds every entry's close-talk
(IHM) wav and its distant-mic (SDM) wavs of those keys, entries lacking a key dropped as the
reference drops them.  Per sample a channel is drawn; the encoder's ``chunk`` is the SDM window
at the IHM chunk's bounds (its tail padded, or the IHM window itself when the SDM ends before
the chunk starts), ``chunk_ctxt`` / ``chunk_rand`` come from SDM wavs of that channel, and
``cchunk``, the targets and the cached slices from the IHM chunk.  Without ``ihm2sdm`` the
dataset feeds IHM data only, as LibriSpeech minus the zero-speech draw.
"""
import json
import os
import pickle
import random
import re

import numpy as np
import torch

from . import ops

FMT_PCM16, FMT_F32 = 0, 1
PLACEMENTS = ("cuda", "pinned", "cpu")
_CR = 6                          # chunk row {fmt, off, L, beg, scale, rbits} (csrc/batch.cu)
_FR = 3                          # frames row {off, frames, s}
_PREFIX = re.compile(r'(\d+).wav')
_NO_TARGET = ("mi", "cmi", "spc", "overlap", "gap", "chunk", "cchunk")
DATASETS = {"LibriSpeechSegTupleWavDataset": "librispeech", "librispeech": "librispeech",
            "AmiSegTupleWavDataset": "ami", "ami": "ami"}


def _channel_keys(ihm2sdm):
    """train.py's ``--ihm2sdm`` ('1,3') or a list of channel keys -> list of str, or None."""
    if ihm2sdm is None:
        return None
    if isinstance(ihm2sdm, str):
        return ihm2sdm.split(',')
    return [str(k) for k in ihm2sdm]


def _place(t, placement, what):
    """Move the host tensor `t` to its placement; 'cuda' is refused when it does not fit."""
    if placement not in PLACEMENTS:
        raise ValueError("%s: placement must be one of %s, got %r" % (what, PLACEMENTS, placement))
    nbytes = t.numel() * t.element_size()
    if placement == "cuda":
        free, _ = torch.cuda.mem_get_info()
        if nbytes > free:
            raise ValueError("%s: %d bytes (%.2f GB) do not fit in the %.2f GB of free device "
                             "memory; use placement='pinned'" % (what, nbytes, nbytes / 1e9,
                                                                 free / 1e9))
        return t.cuda()
    if placement == "pinned":
        return t.pin_memory()
    return t


def _address(t):
    """What the kernels read: the tensor itself (device or, for the emulation, host), or the
    mapped device address of a page-locked host tensor (under UVA, its own address)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr() if t.is_pinned() else t


def read_pool_wav(path):
    """(samples, fmt) of a wav as the pool stores them: PCM16 as int16, float32 as fp32;
    channel 0 of a multi-channel file."""
    from scipy.io import wavfile
    _, data = wavfile.read(path)
    if data.ndim > 1:
        data = data[:, 0]
    if data.dtype == np.int16:
        return np.ascontiguousarray(data), FMT_PCM16
    if data.dtype == np.float32:
        return np.ascontiguousarray(data), FMT_F32
    raise ValueError("%s: %s samples; the corpus pool holds PCM16 and float32 wavs only"
                     % (path, data.dtype))


class WavPool:
    """Every utterance of a split in one buffer per sample format (int16 PCM, fp32), in the
    file order of ``data_cfg[split]['data']``, with int64 offsets and lengths.  A PCM16 sample
    k is read as k * (1 / 32768.f), the value torchaudio.load gives the reference.

    ihm2sdm: AMI channel keys (a list, or train.py's comma-separated string).  Entries that
    lack any of them are dropped, as AmiSegTupleWavDataset drops them (``dropped`` names
    them), and each kept entry's wav under every key is loaded into the same buffers after the
    close-talk wavs.  Files 0..n-1 are the close-talk utterances (``names``); ``channels[key]``
    lists the file of each utterance's distant-mic wav; ``fmt``, ``offs``, ``lens``, ``hold``
    and ``files`` are indexed by file.  A distant-mic file of L samples whose close-talk
    utterance has L' > L + 1 is followed by hold = L' - L - 1 copies of its last sample, the
    most replicate padding its paired window can take (see ``DeviceBatcher._paired``)."""

    def __init__(self, data_root, data_cfg_file, split, placement="cuda", ihm2sdm=None):
        with open(data_cfg_file) as fh:
            cfg = json.load(fh)
        entries = cfg[split]["data"]
        self.ihm2sdm = _channel_keys(ihm2sdm)
        self.dropped = []
        if self.ihm2sdm is not None:
            for key in self.ihm2sdm:
                if not any(key in w for w in entries):
                    raise ValueError("WavPool: channel key %r of ihm2sdm=%s is in no entry of "
                                     "split %r of %s" % (key, ",".join(self.ihm2sdm), split,
                                                         data_cfg_file))
            keep = [all(k in w for k in self.ihm2sdm) for w in entries]
            self.dropped = [w["filename"] for w, k in zip(entries, keep) if not k]
            entries = [w for w, k in zip(entries, keep) if k]
        self.names = [w["filename"] for w in entries]
        if not self.names:
            raise ValueError("WavPool: split %r of %s lists no files" % (split, data_cfg_file))
        self.channels = {}
        self.files = list(self.names)
        for key in dict.fromkeys(self.ihm2sdm or []):
            self.channels[key] = list(range(len(self.files), len(self.files) + len(entries)))
            self.files += [w[key] for w in entries]
        parts = {FMT_PCM16: [], FMT_F32: []}
        fill = {FMT_PCM16: 0, FMT_F32: 0}
        self.fmt, self.offs, self.lens, self.hold = [], [], [], []
        n = len(self.names)
        for f, name in enumerate(self.files):
            x, fmt = read_pool_wav(os.path.join(data_root, name))
            if x.size == 0:
                raise ValueError("WavPool: %s is empty" % name)
            hold = max(0, self.lens[(f - n) % n] - int(x.size) - 1) if f >= n else 0
            self.fmt.append(fmt)
            self.offs.append(fill[fmt])
            self.lens.append(int(x.size))
            self.hold.append(hold)
            parts[fmt].append(x)
            if hold:
                parts[fmt].append(np.full(hold, x[-1], dtype=x.dtype))
            fill[fmt] += int(x.size) + hold
        self.placement = placement
        pcm = np.concatenate(parts[FMT_PCM16]) if parts[FMT_PCM16] else np.zeros(0, np.int16)
        flt = np.concatenate(parts[FMT_F32]) if parts[FMT_F32] else np.zeros(0, np.float32)
        self.pcm = _place(torch.from_numpy(pcm), placement, "WavPool(%s)" % split) \
            if pcm.size else None
        self.flt = _place(torch.from_numpy(flt), placement, "WavPool(%s)" % split) \
            if flt.size else None
        self.index = {n: i for i, n in enumerate(self.names)}

    def __len__(self):
        return len(self.names)

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in (self.pcm, self.flt) if t is not None)

    def samples(self, i):
        """File i (utterance i when i < len(self)) as fp32 numpy (host copy; for tests and
        reports)."""
        t = self.pcm if self.fmt[i] == FMT_PCM16 else self.flt
        x = t[self.offs[i]:self.offs[i] + self.lens[i]].cpu().numpy()
        return x.astype(np.float32) * np.float32(1.0 / 32768) if self.fmt[i] == FMT_PCM16 else x


class FeaturePool:
    """The precomputed ``(F, frames)`` fp32 features of one key for every utterance of the
    pool, read from ``<trans_cache>/<split>/<key>/<basename>.<key>`` (the torch.save files of
    precompute_aco_data.py), concatenated with per-utterance offsets and frame counts."""

    def __init__(self, trans_cache, split, key, names, placement="cuda"):
        self.key = key
        arrays = []
        for name in names:
            base = os.path.splitext(os.path.basename(name))[0]
            path = os.path.join(trans_cache, split, key, base + "." + key)
            if not os.path.exists(path):
                raise ValueError("FeaturePool(%s): cached file %s is missing" % (key, path))
            X = torch.load(path, map_location="cpu")
            if not isinstance(X, torch.Tensor) or X.dim() != 2 or X.dtype != torch.float32:
                raise ValueError("FeaturePool(%s): %s holds %s, expected a 2-D float32 tensor"
                                 % (key, path, getattr(X, "dtype", type(X))))
            if arrays and X.shape[0] != arrays[0].shape[0]:
                raise ValueError("FeaturePool(%s): %s has F=%d, the first file has F=%d"
                                 % (key, path, X.shape[0], arrays[0].shape[0]))
            arrays.append(X.contiguous())
        self.F = int(arrays[0].shape[0])
        self.frames = [int(a.shape[1]) for a in arrays]
        self.offs = np.concatenate([[0], np.cumsum([a.numel() for a in arrays])[:-1]]) \
            .astype(np.int64).tolist()
        flat = torch.cat([a.reshape(-1) for a in arrays])
        self.placement = placement
        self.data = _place(flat, placement, "FeaturePool(%s)" % key)

    def nbytes(self):
        return self.data.numel() * 4


class SamplePlan(dict):
    """One sample's draws: index, ctxt, rand, beg (per source), scale (per source, or None),
    slices (key -> first frame), distortions (the Distortions draw dict)."""


class BatchPlan:
    """Draws of one batch: ``samples[b]`` the per-sample draws, ``table`` the packed int64
    vector the kernels read (float fields bit-cast), ``offsets`` its sections."""

    def __init__(self, B, T, samples, table, offsets, dist_plan):
        self.B, self.T, self.samples, self.table = B, T, samples, table
        self.offsets, self.dist_plan = offsets, dist_plan


class DeviceBatcher:
    """Assembles collated PASE+ training batches on the device from a :class:`WavPool`.

    chunk_size: T.  mi: MIChunkWav (chunk, chunk_ctxt, chunk_rand) else SingleChunkWav.
    cached: {key: (FeaturePool, hop)}, gathered and not z-normed.  targets: device
    :class:`pase_b200.targets.LPS` objects run on the clean chunk.  distortions: a
    :class:`pase_b200.distortions.Distortions` applied to ``chunk``.  order: the target
    names in the reference's transform order (default: targets, then cached keys); the hop
    of the last one sets the overlap label's resolution.  dataset: 'librispeech' or 'ami' (or
    the reference's class names).  ihm2sdm: for 'ami', the channel keys to pair with, the
    ones the pool was loaded with; None feeds close-talk data only.
    """

    def __init__(self, wav_pool, chunk_size, mi=True, random_scale=False, cached=None,
                 targets=None, distortions=None, zero_speech_p=0, order=None,
                 dataset="librispeech", ihm2sdm=None):
        if dataset not in DATASETS:
            raise ValueError("DeviceBatcher: dataset %r is not assembled on the device; one of %s"
                             % (dataset, sorted(DATASETS)))
        self.dataset = DATASETS[dataset]
        self.ihm2sdm = _channel_keys(ihm2sdm)
        if self.dataset == "ami":
            if zero_speech_p > 0:
                raise ValueError("DeviceBatcher: AmiSegTupleWavDataset has no zero-speech "
                                 "samples; zero_speech_p=%g must be 0" % zero_speech_p)
            if self.ihm2sdm != wav_pool.ihm2sdm:
                raise ValueError("DeviceBatcher: ihm2sdm=%s, the pool was loaded with ihm2sdm=%s"
                                 % (self.ihm2sdm, wav_pool.ihm2sdm))
        elif self.ihm2sdm is not None or wav_pool.ihm2sdm is not None:
            raise ValueError("DeviceBatcher: ihm2sdm pairs channels of the 'ami' dataset only; "
                             "LibriSpeechSegTupleWavDataset reads close-talk files")
        if zero_speech_p > 0:
            raise NotImplementedError("DeviceBatcher: zero_speech_p=%g > 0 (zero-speech "
                                      "samples) is not supported; set it to 0" % zero_speech_p)
        if len(wav_pool) < 2:
            raise ValueError("DeviceBatcher: the random utterance needs at least 2 utterances, "
                             "the pool has %d" % len(wav_pool))
        T = int(chunk_size)
        if T < 2:
            raise ValueError("DeviceBatcher: chunk_size=%d" % T)
        self.wavs, self.T, self.mi, self.random_scale = wav_pool, T, bool(mi), bool(random_scale)
        self.cached = dict(cached or {})
        self.targets = list(targets or [])
        self.distortions = distortions
        self.zero_speech_p = zero_speech_p
        for key, (pool, hop) in self.cached.items():
            if T % hop != 0:
                raise ValueError("DeviceBatcher: cached key '%s': chunk_size %d is not a multiple "
                                 "of hop %d, so the frame slices would differ in length"
                                 % (key, T, hop))
            if len(pool.frames) != len(wav_pool):
                raise ValueError("DeviceBatcher: cached key '%s' has %d utterances, the pool %d"
                                 % (key, len(pool.frames), len(wav_pool)))
        hops = {t.name: t.hop for t in self.targets}
        hops.update({k: h for k, (_, h) in self.cached.items()})
        self.order = list(order) if order is not None else list(hops)
        self.d = hops[self.order[-1]] if self.order else 1
        if T % self.d != 0:
            raise ValueError("DeviceBatcher: chunk_size %d is not a multiple of the label "
                             "resolution %d" % (T, self.d))
        self.nsrc = 3 if self.mi else 1
        self.paired = self.ihm2sdm is not None
        self._dist_offsets = {}
        self.reset()

    # ---- construction from train.py's options --------------------------------------------
    @classmethod
    def from_train_opts(cls, workers_cfg, chunk_size, hop, wav_pool, random_scale=False,
                        stats=None, trans_cache=None, split="train", distortions=None,
                        feature_placement="cuda", device="cuda",
                        dataset="LibriSpeechSegTupleWavDataset", ihm2sdm=None):
        """The transforms train.py:37-136 (make_transforms) builds from a workers cfg (a dict
        or a json path): every key with a cache directory is gathered from a FeaturePool, an
        lps* key without one becomes a device LPS with its stats folded in as ZNorm, any other
        target key without one raises NotImplementedError.  dataset, ihm2sdm: train.py's
        ``--dataset`` (a name, or its list of one) and ``--ihm2sdm``; the cached features of
        an AMI pool are the close-talk utterances'."""
        from .targets import LPS
        if isinstance(dataset, (list, tuple)):
            if len(dataset) != 1:
                raise NotImplementedError("DeviceBatcher: %d datasets %s; a concatenation of "
                                          "datasets (MetaWavConcatDataset) is not assembled on "
                                          "the device" % (len(dataset), list(dataset)))
            dataset = dataset[0]
        if dataset not in DATASETS:
            raise ValueError("DeviceBatcher: dataset %r is not assembled on the device; one of %s"
                             % (dataset, sorted(DATASETS)))
        if isinstance(workers_cfg, str):
            with open(workers_cfg) as fh:
                workers_cfg = json.load(fh)
        mi = any("mi" in m["name"] for ms in workers_cfg.values() for m in ms)
        st = None
        if stats is not None:
            with open(stats, "rb") as fh:
                st = pickle.load(fh)
        seen, cached, targets, order = [], {}, [], []
        for ms in workers_cfg.values():
            for m in ms:
                name = m["name"]
                if name in seen:
                    raise ValueError("Duplicated key {} in minions".format(name))
                seen.append(name)
                tr = dict(m.get("transform", {}))
                tr["hop"] = hop
                if name in _NO_TARGET or "regu" in name:
                    continue
                if trans_cache is not None and os.path.isdir(os.path.join(trans_cache, split, name)):
                    cached[name] = (FeaturePool(trans_cache, split, name, wav_pool.names,
                                                feature_placement), hop)
                elif "lps" in name:
                    s = None
                    if st is not None and name in st:
                        s = (st[name]["mean"], st[name]["std"])
                    tr["name"] = name
                    targets.append(LPS(device=device, stats=s, **tr))
                else:
                    raise NotImplementedError(
                        "DeviceBatcher: target '%s' has no feature cache (%s) and cannot be "
                        "computed on the device; precompute it with precompute_aco_data.py"
                        % (name, os.path.join(str(trans_cache), split, name)))
                order.append(name)
        return cls(wav_pool, chunk_size, mi=mi, random_scale=random_scale, cached=cached,
                   targets=targets, distortions=distortions, order=order, dataset=dataset,
                   ihm2sdm=ihm2sdm)

    # ---- host planner --------------------------------------------------------------------
    def reset(self):
        """Restore the neighbour lists (what a new epoch's freshly forked loader sees)."""
        self._neighbors = {}
        for name in self.wavs.names:
            self._neighbors.setdefault(_PREFIX.sub('', name), []).append(name)

    def _window(self, i, npr):
        L, T = self.wavs.lens[i], self.T
        if L > T:
            return int(npr.randint(0, L - T))
        if T - L >= L:
            raise ValueError("utterance %s: %d samples cannot be reflect-padded to chunk_size "
                             "%d (padding %d >= length)" % (self.wavs.files[i], L, T, T - L))
        return 0

    def _paired(self, f, beg):
        """select_chunk(sdm, reuse_bounds=(beg, beg + T)) of file f: (beg, pad) with pad one of
        'whole' (the file reflect-padded from 0), 'slice', 'reflect' or 'replicate' (the tail
        from beg padded), or None when beg is past its end (the chunk then stands in for it).
        Each is a plain chunk row: the reflected tail as a file of its own that starts at beg,
        the replicated tail as a slice running into the copies of the last sample the pool
        holds after the file.  The replicate padding P = T - (L - beg) fits in them: the IHM
        window start is at most L' - T - 1, so P <= L' - L - 1."""
        L, T = self.wavs.lens[f], self.T
        if L <= T:                                  # the whole file, reflect-padded from 0
            if T - L >= L:
                raise ValueError("distant-mic file %s: %d samples cannot be reflect-padded to "
                                 "chunk_size %d (padding %d >= length)"
                                 % (self.wavs.files[f], L, T, T - L))
            return 0, "whole"
        if beg + T <= L:
            return beg, "slice"
        if beg >= L:
            return None
        n = L - beg                                 # the tail, reflected when F.pad can
        if T - n < n:
            return beg, "reflect"
        if T - n > self.wavs.hold[f]:
            raise ValueError("distant-mic file %s: the window at %d needs %d samples of "
                             "replicate padding, the pool holds %d"
                             % (self.wavs.files[f], beg, T - n, self.wavs.hold[f]))
        return beg, "replicate"

    def _draw_ami(self, index, py, npr):
        """One sample's utterances and windows, in the order AmiSegTupleWavDataset.__getitem__
        and MIChunkWav / SingleChunkWav draw them."""
        W, n = self.wavs, len(self.wavs)
        name = W.names[index]
        nb = self._neighbors[_PREFIX.sub('', name)]
        if name not in nb:
            raise ValueError("utterance %d (%s) visited twice before reset()" % (index, name))
        nb.remove(name)
        ctxt = W.index[py.choice(nb)] if nb else index
        j = py.choice(range(n - 1))                 # = choice(indices without index)
        rand = j + (j >= index)
        s = SamplePlan(index=index, ctxt=ctxt, rand=rand)
        files = (index, ctxt, rand)
        if self.paired:
            s["channel"] = py.choice(self.ihm2sdm)
            sdm = W.channels[s["channel"]]
            files = (index, sdm[ctxt], sdm[rand])
        s["files"] = files if self.mi else files[:1]
        s["beg"] = [self._window(index, npr)]
        if self.paired:
            s["paired"] = self._paired(sdm[index], s["beg"][0])
        s["beg"] += [self._window(f, npr) for f in s["files"][1:]]
        return s

    def _draw(self, index, py, npr, tg):
        """One sample, in the order LibriSpeechSegTupleWavDataset.__getitem__ draws (or
        AmiSegTupleWavDataset's: no zero-speech coin, a channel after the random utterance)."""
        names, n = self.wavs.names, len(self.wavs)
        if not 0 <= index < n:
            raise ValueError("index %d outside the pool of %d utterances" % (index, n))
        if self.dataset == "ami":
            s = self._draw_ami(index, py, npr)
            beg, nscale = s["beg"], len(s["files"]) + self.paired   # the paired cchunk last
        else:
            py.random() < self.zero_speech_p        # sample_probable: drawn even when p = 0
            name = names[index]
            nb = self._neighbors[_PREFIX.sub('', name)]
            if name not in nb:
                raise ValueError("utterance %d (%s) visited twice before reset()" % (index, name))
            nb.remove(name)
            ctxt = self.wavs.index[py.choice(nb)] if nb else index
            j = py.choice(range(n - 1))             # = choice(indices without index)
            rand = j + (j >= index)
            srcs = (index, ctxt, rand) if self.mi else (index,)
            beg = [self._window(i, npr) for i in srcs]
            s = SamplePlan(index=index, ctxt=ctxt, rand=rand, beg=beg)
            nscale = len(srcs)
        name = names[index]
        scale = None
        if self.random_scale:
            scale = [float(torch.rand(1, generator=tg)) for _ in range(nscale)]
        s.update(scale=scale, slices={})
        for key, (pool, hop) in self.cached.items():
            a, e = beg[0] // hop, (beg[0] + self.T) // hop
            if e > pool.frames[index]:
                raise ValueError("cached key '%s': utterance %s has %d frames, the chunk at %d "
                                 "needs frames [%d, %d)" % (key, name, pool.frames[index],
                                                            beg[0], a, e))
            s["slices"][key] = a
        if self.distortions is not None:
            s["distortions"] = self.distortions._draw(self.T, py, npr)
        return s

    def plan(self, indices, rng=None):
        """Draw the plan of the batch `indices`.  rng: None (the global random, np.random and
        torch's default generator) or (random.Random, np.random.RandomState, torch.Generator)."""
        indices = [int(i) for i in indices]
        if not indices:
            raise ValueError("plan: empty batch")
        py, npr, tg = (random, np.random, None) if rng is None else rng
        samples = [self._draw(i, py, npr, tg) for i in indices]
        return self._pack(samples)

    def _layout(self, B):
        offs, o = {"chunk": (0, self.nsrc * _CR)}, B * self.nsrc * _CR
        if self.paired:                             # the close-talk rows, gathered into cchunk
            offs["cchunk"] = (o, _CR)
            o += B * _CR
        for key in self.cached:
            offs[key] = (o, _FR)
            o += B * _FR
        return offs, o

    def _dist_offsets_for(self, B):
        if B not in self._dist_offsets:
            self._dist_offsets[B] = self.distortions._pack(B, self.T, [{}] * B)
        return self._dist_offsets[B]

    def _pack(self, samples):
        B, T, W = len(samples), self.T, self.wavs
        offs, n = self._layout(B)
        dist_plan = None
        if self.distortions is not None:
            dist_plan = self.distortions._pack(B, T, [s["distortions"] for s in samples])
            offs["dist"] = (n, dist_plan.table.size)
            n += dist_plan.table.size
        table = np.zeros(n, dtype=np.int64)
        crow = table[:B * self.nsrc * _CR].reshape(B, self.nsrc, _CR)

        def row(s, i, beg, k, pad="slice"):
            rbits = 0
            if s["scale"] is not None:
                rbits = int(np.array(s["scale"][k], np.float32).view(np.int32))
            off, L = W.offs[i], W.lens[i]
            if pad == "reflect":                    # the tail as a file of its own
                off, L, beg = off + beg, L - beg, 0
            elif pad == "replicate":                # into the copies of the last sample
                L += W.hold[i]
            return (W.fmt[i], off, L, beg, 1 if s["scale"] is not None else 0, rbits)

        for b, s in enumerate(samples):
            srcs = s.get("files") or ((s["index"], s["ctxt"], s["rand"]) if self.mi
                                      else (s["index"],))
            rows = [row(s, i, s["beg"][k], k) for k, i in enumerate(srcs)]
            if self.paired:
                # cchunk: the close-talk window with the first scale draw; chunk: the
                # distant-mic window, or the close-talk window itself, with the last
                a = offs["cchunk"][0] + b * _CR
                table[a:a + _CR] = rows[0]
                p, k = s["paired"], len(srcs)
                sdm = self.wavs.channels[s["channel"]][s["index"]]
                rows[0] = row(s, s["index"], s["beg"][0], k) if p is None else \
                    row(s, sdm, p[0], k, p[1])
            crow[b] = rows
            for key, (pool, _) in self.cached.items():
                a = offs[key][0]
                table[a + b * _FR:a + (b + 1) * _FR] = (pool.offs[s["index"]],
                                                        pool.frames[s["index"]], s["slices"][key])
        if dist_plan is not None:
            table[offs["dist"][0]:] = dist_plan.table
        return BatchPlan(B, T, samples, table, offs, dist_plan)

    # ---- device side ---------------------------------------------------------------------
    def upload(self, plan, out=None):
        """Copy the plan table to the device (one H2D copy); into `out` when given (a graph
        replays with a newly uploaded plan this way)."""
        src = torch.from_numpy(plan.table)
        dev = self._device()
        if dev.type == "cuda":
            src = src.pin_memory()
        if out is None:
            return src.to(dev, non_blocking=True)
        if out.numel() != src.numel() or out.dtype != torch.int64:
            raise ValueError("upload: table of %d int64 expected, got %d %s"
                             % (src.numel(), out.numel(), out.dtype))
        out.copy_(src, non_blocking=True)
        return out

    def _device(self):
        for t in (self.wavs.pcm, self.wavs.flt):
            if t is not None:
                return torch.device("cuda") if t.is_pinned() else t.device
        return torch.device("cuda")

    def _batch_size(self, table):
        w = (self.nsrc + self.paired) * _CR + _FR * len(self.cached)
        if self.distortions is not None:
            w += self._dist_offsets_for(1).table.size
        if table.numel() % w:
            raise ValueError("run: a table of %d int64 is not a whole batch of %d-entry rows"
                             % (table.numel(), w))
        return table.numel() // w

    def run(self, table):
        """The collated batch of the device plan `table`: chunk windows, targets on the clean
        chunk, cached slices, the overlap label, then the distortions of chunk in place.  Launch
        shapes depend only on (B, T, configuration)."""
        B, T = self._batch_size(table), self.T
        offs, _ = self._layout(B)
        dev = table.device
        nout = self.nsrc + 1
        buf = torch.empty((nout, B, 1, T), dtype=torch.float32, device=dev)
        W = self.wavs
        pcm, flt = _address(W.pcm), _address(W.flt)
        npcm, nflt = 0 if pcm is None else W.pcm.numel(), 0 if flt is None else W.flt.numel()
        ops.call("pase_chunk_gather", pcm, npcm, flt, nflt, table[:B * self.nsrc * _CR], B,
                 self.nsrc, T, 0 if self.paired else 1, buf, B * T)
        if self.paired:
            a = offs["cchunk"][0]
            ops.call("pase_chunk_gather", pcm, npcm, flt, nflt, table[a:a + B * _CR], B, 1, T, 0,
                     buf[self.nsrc], B * T)
        out = {"chunk": buf[0], "cchunk": buf[self.nsrc]}
        if self.mi:
            out["chunk_ctxt"], out["chunk_rand"] = buf[1], buf[2]
        for t in self.targets:
            out[t.name] = t(out["cchunk"])
        for key, (pool, hop) in self.cached.items():
            a = offs[key][0]
            n = T // hop
            y = torch.empty((B, pool.F, n), dtype=torch.float32, device=dev)
            ops.call("pase_frames_gather", _address(pool.data), pool.data.numel(),
                     table[a:a + B * _FR], B, pool.F, n, y)
            out[key] = y
        lab = torch.empty((B, 1, T // self.d), dtype=torch.float32, device=dev)
        if self.distortions is not None:
            a = B * (self.nsrc + self.paired) * _CR + B * _FR * len(self.cached)
            self.distortions.run(out["chunk"].view(B, T), table[a:],
                                 self._dist_offsets_for(B).offsets, lab.view(B, -1), self.d)
        else:
            lab.zero_()
        out["overlap"] = lab
        return out

    def __call__(self, indices, rng=None):
        return self.run(self.upload(self.plan(indices, rng)))
