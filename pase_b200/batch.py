"""On-device batch assembly: a drop-in for the reference's DataLoader over
``LibriSpeechSegTupleWavDataset`` (pase/dataset.py:428-513) with ``MIChunkWav`` /
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
    k is read as k * (1 / 32768.f), the value torchaudio.load gives the reference."""

    def __init__(self, data_root, data_cfg_file, split, placement="cuda"):
        with open(data_cfg_file) as fh:
            cfg = json.load(fh)
        self.names = [w["filename"] for w in cfg[split]["data"]]
        if not self.names:
            raise ValueError("WavPool: split %r of %s lists no files" % (split, data_cfg_file))
        parts = {FMT_PCM16: [], FMT_F32: []}
        fill = {FMT_PCM16: 0, FMT_F32: 0}
        self.fmt, self.offs, self.lens = [], [], []
        for name in self.names:
            x, fmt = read_pool_wav(os.path.join(data_root, name))
            if x.size == 0:
                raise ValueError("WavPool: %s is empty" % name)
            self.fmt.append(fmt)
            self.offs.append(fill[fmt])
            self.lens.append(int(x.size))
            parts[fmt].append(x)
            fill[fmt] += int(x.size)
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
        """Utterance i as fp32 numpy (host copy; for tests and reports)."""
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
    of the last one sets the overlap label's resolution.
    """

    def __init__(self, wav_pool, chunk_size, mi=True, random_scale=False, cached=None,
                 targets=None, distortions=None, zero_speech_p=0, order=None):
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
        self._dist_offsets = {}
        self.reset()

    # ---- construction from train.py's options --------------------------------------------
    @classmethod
    def from_train_opts(cls, workers_cfg, chunk_size, hop, wav_pool, random_scale=False,
                        stats=None, trans_cache=None, split="train", distortions=None,
                        feature_placement="cuda", device="cuda"):
        """The transforms train.py:37-136 (make_transforms) builds from a workers cfg (a dict
        or a json path): every key with a cache directory is gathered from a FeaturePool, an
        lps* key without one becomes a device LPS with its stats folded in as ZNorm, any other
        target key without one raises NotImplementedError."""
        from .targets import LPS
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
                   targets=targets, distortions=distortions, order=order)

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
                             "%d (padding %d >= length)" % (self.wavs.names[i], L, T, T - L))
        return 0

    def _draw(self, index, py, npr, tg):
        """One sample, in the order LibriSpeechSegTupleWavDataset.__getitem__ draws."""
        names, n = self.wavs.names, len(self.wavs)
        if not 0 <= index < n:
            raise ValueError("index %d outside the pool of %d utterances" % (index, n))
        py.random() < self.zero_speech_p            # sample_probable: drawn even when p = 0
        name = names[index]
        nb = self._neighbors[_PREFIX.sub('', name)]
        if name not in nb:
            raise ValueError("utterance %d (%s) visited twice before reset()" % (index, name))
        nb.remove(name)
        ctxt = self.wavs.index[py.choice(nb)] if nb else index
        j = py.choice(range(n - 1))                 # = choice(indices without index)
        rand = j + (j >= index)
        srcs = (index, ctxt, rand) if self.mi else (index,)
        beg = [self._window(i, npr) for i in srcs]
        scale = None
        if self.random_scale:
            scale = [float(torch.rand(1, generator=tg)) for _ in srcs]
        s = SamplePlan(index=index, ctxt=ctxt, rand=rand, beg=beg, scale=scale, slices={})
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
        for b, s in enumerate(samples):
            srcs = (s["index"], s["ctxt"], s["rand"]) if self.mi else (s["index"],)
            for k, i in enumerate(srcs):
                rbits = 0
                if s["scale"] is not None:
                    rbits = int(np.array(s["scale"][k], np.float32).view(np.int32))
                crow[b, k] = (W.fmt[i], W.offs[i], W.lens[i], s["beg"][k],
                              1 if s["scale"] is not None else 0, rbits)
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
        w = self.nsrc * _CR + _FR * len(self.cached)
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
        ops.call("pase_chunk_gather", pcm, 0 if pcm is None else W.pcm.numel(), flt,
                 0 if flt is None else W.flt.numel(), table[:B * self.nsrc * _CR], B, self.nsrc,
                 T, 1, buf, B * T)
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
            a = B * self.nsrc * _CR + B * _FR * len(self.cached)
            self.distortions.run(out["chunk"].view(B, T), table[a:],
                                 self._dist_offsets_for(B).offsets, lab.view(B, -1), self.d)
        else:
            lab.zero_()
        out["overlap"] = lab
        return out

    def __call__(self, indices, rng=None):
        return self.run(self.upload(self.plan(indices, rng)))
