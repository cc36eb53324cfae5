"""On-device PASE+ waveform distortions: a drop-in for the reference's
``pase.transforms.config_distortions(...)`` / ``PCompose`` (pase/transforms.py:38-146) that
works on a collated batch already in HBM.

    dist = config_distortions(**json.load(open('cfg/distortions/pase+.cfg')), codec2_p=0)
    batch = {k: v.to(dev) for k, v in batch.items()}
    ... compute the targets from the clean batch['chunk'] ...
    dist(batch)        # batch['chunk'] <- distorted copy, batch['overlap'] <- overlap label

Per sample b = 0..B-1 the host draws from Python ``random`` and numpy's global ``np.random``
exactly as the reference's PCompose would for that sample (or from an explicit
``(random.Random, np.random.RandomState)`` pair), then the stages run as CUDA kernels
(pase_b200/csrc/distort.cu) that read which samples they touch from one uploaded plan table.
Supported stages, in the reference's order: Reverb, SimpleAdditiveShift (overlap), SimpleAdditive
(noise), Clipping, BandDrop, Downsample.  codec2, chop, speed and resample raise
NotImplementedError: nothing is silently skipped.

Differences from the reference: an IR whose peak is its first tap (p = 0), and a 1-tap FIR
(shift round(1/2) = 0), make the reference's ``shift(xs, 0)`` fail; here that shift is the
identity.  The convolutions run in fp32 through FFTs (DESIGN.md section 10); energies are
accumulated in fp64.
"""
import ctypes
import glob
import os
import random

import numpy as np
import torch

from . import ops

BLOCK = 4096                      # overlap-save block and filter partition (distort.cu)
MAX_REVERB_LEN = 24000            # Reverb(max_reverb_len) default, transforms.py:1004
STAGES = ("reverb", "overlap", "noise", "clip", "bandrop", "downsample")

# plan table: per stage a (B, width) int64 block, then (B,) float64 vectors; section order fixed
_INT_SECTIONS = (("rev", 6), ("ovseg", 3), ("ovrev", 6), ("ovmix", 3), ("nseg", 3),
                 ("nmix", 3), ("clip", 1), ("bd", 6), ("ds", 6))
_DBL_SECTIONS = ("ovsnr", "nsnr", "cf")


def _twiddles():
    k = np.arange(BLOCK, dtype=np.float64)
    w = np.exp(-2j * np.pi * k / (2 * BLOCK))
    return np.stack([w.real, w.imag], axis=1).astype(np.float32).reshape(-1)


def read_wav(path):
    """Samples of a mono wav as float64, the values soundfile.read returns: soundfile when it
    is importable, otherwise scipy's reader for PCM16 (/ 32768) and float wavs."""
    try:
        import soundfile as sf
    except ImportError:
        sf = None
    if sf is not None:
        data, _ = sf.read(path)
    else:
        from scipy.io import wavfile
        _, data = wavfile.read(path)
        if data.dtype == np.int16:
            data = data.astype(np.float64) / 32768.0
        elif data.dtype in (np.float32, np.float64):
            data = data.astype(np.float64)
        else:
            raise RuntimeError("%s: %s samples need the soundfile package (only PCM16 and float "
                               "wavs are read without it)" % (path, data.dtype))
    if data.ndim != 1:
        raise ValueError("%s: expected a mono wav, got shape %s" % (path, data.shape))
    return data


def load_ir(path, fmt):
    """Reverb.load_IR (transforms.py:1028-1051): raw IR as float64."""
    if fmt == "mat":
        from scipy.io import loadmat
        return np.asarray(loadmat(path, squeeze_me=True, struct_as_record=False)["risp_imp"],
                          dtype=np.float64).reshape(-1)
    if fmt in ("imp", "txt"):
        return np.loadtxt(path).astype(np.float64).reshape(-1)
    if fmt == "npy":
        return np.load(path).astype(np.float64).reshape(-1)
    if fmt == "wav":
        return read_wav(path)
    raise TypeError("Unrecognized IR format: %s" % fmt)


def load_filter(path, fmt):
    """BandDrop / Downsample.load_filter (transforms.py:1226-1243): raw taps as float64."""
    if fmt == "mat":
        from scipy.io import loadmat
        return np.asarray(loadmat(path, squeeze_me=True, struct_as_record=False)["filt_coeff"],
                          dtype=np.float64).reshape(-1)
    if fmt in ("imp", "txt"):
        return np.loadtxt(path).astype(np.float64).reshape(-1)
    if fmt == "npy":
        return np.load(path).astype(np.float64).reshape(-1)
    raise TypeError("Unrecognized filter format: %s" % fmt)


class _Bank:
    """Filters concatenated into one device fp32 vector: offsets, lengths, shifts."""

    def __init__(self, names, arrays, shifts, device):
        self.names = list(names)
        self.lens = [len(a) for a in arrays]
        self.offs = np.concatenate([[0], np.cumsum(self.lens)[:-1]]).astype(np.int64).tolist()
        self.shifts = list(shifts)
        self.lmax = max(self.lens)
        flat = np.concatenate(arrays).astype(np.float32)
        self.data = torch.from_numpy(flat).to(device)

    def __len__(self):
        return len(self.names)


def _ir_bank(files, root, fmt, device):
    arrays, shifts = [], []
    for f in files:
        h = load_ir(os.path.join(root, f), fmt)[:MAX_REVERB_LEN]
        if h.size == 0:
            raise ValueError("empty IR %s" % f)
        if np.max(h) > 0:
            h = h / np.abs(np.max(h))
        arrays.append(h)
        shifts.append(int(np.argmax(np.abs(h))))
    return _Bank(files, arrays, shifts, device)


def _fir_bank(files, root, fmt, device):
    arrays, shifts = [], []
    for f in files:
        c = load_filter(os.path.join(root, f), fmt)
        if c.size == 0:
            raise ValueError("empty filter %s" % f)
        c = c / np.abs(np.max(c))
        arrays.append(c)
        shifts.append(int(round(c.shape[0] / 2)))        # Python round: half to even
    return _Bank(files, arrays, shifts, device)


def _noise_bank(paths, device):
    arrays = [read_wav(p) for p in paths]
    for p, a in zip(paths, arrays):
        if a.size == 0:
            raise ValueError("empty noise file %s" % p)
    return _Bank(paths, arrays, [0] * len(paths), device)


def _glob_files(root, fmt):
    return [os.path.basename(f) for f in glob.glob(os.path.join(root, "*.{}".format(fmt)))]


def _noise_paths(dirs, listfile=None):
    if listfile is not None:
        if isinstance(dirs, list):
            assert len(dirs) == 1, len(dirs)
            dirs = dirs[0]
        with open(listfile) as fh:
            return [os.path.join(dirs, line.rstrip()) for line in fh]
    if isinstance(dirs, list):
        out = []
        for d in dirs:
            out += glob.glob(os.path.join(d, "*.wav"))
        return out
    return glob.glob(os.path.join(dirs, "*.wav"))


class DistortionPlan:
    """Per-sample draws of one batch: ``samples[b]`` maps each applied stage to its choices,
    ``table`` is the packed int64 vector the kernels read (float64 fields bit-cast)."""

    def __init__(self, B, T, samples, table, offsets):
        self.B, self.T, self.samples, self.table, self.offsets = B, T, samples, table, offsets


class Distortions:
    """Device replacement of the reference's PCompose of distortions.  Construct it with
    :func:`config_distortions`.

    Memory: every IR, FIR and noise / overlap wav is loaded once into device memory as fp32,
    4 bytes per sample (IRs truncated to 24000 taps).  A call allocates, through torch's
    caching allocator, the distorted copy and one segment buffer (4 B T bytes each) and, per
    convolution stage, a workspace of 64 KB x B x (ceil((T + Lmax - 1) / 4096) +
    ceil(Lmax / 4096)) plus 4 B T bytes (Lmax = the bank's longest filter): about 100 MB
    for a 24000-tap IR bank at B = 64, T = 48000.
    """

    def __init__(self, cfg, device):
        self.device = torch.device(device)
        self.report = bool(cfg.get("report", False))
        self.stages = []                       # (name, p)
        self.ir = self.ov = self.noise = self.bd = self.ds = None
        c = cfg
        rev_files = c["reverb_irfiles"]
        need_rev = (c["reverb_p"] > 0 and rev_files is not None) or \
            (c["overlap_p"] > 0 and c["overlap_dir"] is not None and c["overlap_reverb"])
        if need_rev:
            if rev_files is None:
                raise ValueError("overlap_reverb needs reverb_irfiles")
            if len(rev_files) == 0:
                rev_files = _glob_files(c["reverb_data_root"], c["reverb_fmt"])
            if len(rev_files) == 0:
                raise ValueError("no *.%s IR files in %s" % (c["reverb_fmt"], c["reverb_data_root"]))
            self.ir = _ir_bank(rev_files, c["reverb_data_root"], c["reverb_fmt"], self.device)
        if c["reverb_p"] > 0 and c["reverb_irfiles"] is not None:
            self.stages.append(("reverb", c["reverb_p"]))
        if c["overlap_p"] > 0 and c["overlap_dir"] is not None:
            paths = _noise_paths(c["overlap_dir"], c["overlap_list"])
            if len(paths) == 0:
                raise ValueError("[!] No noises found in {}".format(c["overlap_dir"]))
            self.ov = _noise_bank(paths, self.device)
            self.ov_snrs = list(c["overlap_snrs"])
            self.ov_reverb = bool(c["overlap_reverb"])
            self.stages.append(("overlap", c["overlap_p"]))
        if c["noises_p"] > 0 and c["noises_dir"] is not None:
            paths = _noise_paths(c["noises_dir"])
            if len(paths) == 0:
                raise ValueError("[!] No noises found in {}".format(c["noises_dir"]))
            self.noise = _noise_bank(paths, self.device)
            self.noise_snrs = list(c["noises_snrs"])
            self.stages.append(("noise", c["noises_p"]))
        if c["clip_p"] > 0 and len(c["clip_factors"]) > 0:
            self.clip_factors = list(c["clip_factors"])
            self.stages.append(("clip", c["clip_p"]))
        if c["bandrop_p"] > 0 and c["bandrop_irfiles"] is not None:
            files = c["bandrop_irfiles"]
            if len(files) == 0:
                files = _glob_files(c["bandrop_data_root"], c["bandrop_fmt"])
            if len(files) == 0:
                raise ValueError("no *.%s filters in %s" % (c["bandrop_fmt"], c["bandrop_data_root"]))
            self.bd = _fir_bank(files, c["bandrop_data_root"], c["bandrop_fmt"], self.device)
            self.stages.append(("bandrop", c["bandrop_p"]))
        if c["downsample_p"] > 0 and len(c["downsample_irfiles"]) > 0:
            self.ds = _fir_bank(c["downsample_irfiles"], c["downsample_data_root"],
                                c["downsample_fmt"], self.device)
            self.stages.append(("downsample", c["downsample_p"]))
        self.twiddle = torch.from_numpy(_twiddles()).to(self.device) if self.stages else None

    def __repr__(self):
        return "Distortions(%s)" % ", ".join("%s p=%g" % s for s in self.stages)

    # ---- host planner ----------------------------------------------------------------
    def _draw(self, T, py, npr):
        """One sample's draws, in the reference's order (transforms.py:84-141, 221-233)."""
        s = {}
        for name, p in self.stages:
            if not py.random() < p:
                continue
            if name == "reverb":
                s["reverb"] = {"ir": py.choice(list(range(len(self.ir))))}
            elif name == "overlap":
                shift = int(npr.randint(0, int(0.75 * T)))
                nf = len(self.ov)
                f = int(npr.randint(0, nf)) if nf > 1 else 0
                Ts, Lf = T - shift, self.ov.lens[f]
                beg = int(npr.randint(0, Lf - Ts)) if Lf > Ts else 0
                d = {"shift": shift, "file": f, "beg": beg}
                if self.ov_reverb:
                    d["ir"] = py.choice(list(range(len(self.ir))))
                d["snr"] = py.choice(self.ov_snrs)
                s["overlap"] = d
            elif name == "noise":
                nf = len(self.noise)
                f = int(npr.randint(0, nf)) if nf > 1 else 0
                Lf = max(self.noise.lens[f], T)
                beg = int(npr.randint(0, Lf - T)) if Lf > T else 0
                s["noise"] = {"file": f, "beg": beg, "snr": py.choice(self.noise_snrs)}
            elif name == "clip":
                s["clip"] = {"cf": py.choice(self.clip_factors)}
            else:
                bank = self.bd if name == "bandrop" else self.ds
                s[name] = {"filt": py.choice(list(range(len(bank))))}
        return s

    def plan(self, B, T, rng=None):
        """Draw the plan of a (B, 1, T) batch.  rng: None (the global ``random`` and
        ``np.random``, as the reference's DataLoader workers) or (random.Random,
        np.random.RandomState)."""
        if B < 1 or T < 2:
            raise ValueError("plan: need B >= 1 and T >= 2, got B=%d T=%d" % (B, T))
        py, npr = (random, np.random) if rng is None else rng
        samples = [self._draw(T, py, npr) for _ in range(B)]
        return self._pack(B, T, samples)

    def _pack(self, B, T, samples):
        offs, o = {}, 0
        for name, w in _INT_SECTIONS:
            offs[name] = (o, w)
            o += B * w
        for name in _DBL_SECTIONS:
            offs[name] = (o, 1)
            o += B
        table = np.zeros(o, dtype=np.int64)
        sec = {n: table[a:a + B * w].reshape(B, w) for n, (a, w) in offs.items()
               if n not in _DBL_SECTIONS}
        dbl = {n: table[offs[n][0]:offs[n][0] + B].view(np.float64) for n in _DBL_SECTIONS}

        def conv_row(row, bank, i, n, mode):
            L, off, p = bank.lens[i], bank.offs[i], bank.shifts[i]
            if not (0 <= i < len(bank) and 0 < n <= T and 0 <= p < L and
                    off + L <= bank.data.numel()):
                raise ValueError("plan: filter %d (L=%d, p=%d) does not fit its bank" % (i, L, p))
            row[:] = (1, n, off, L, p, mode)

        def seg_row(row, bank, f, beg, n):
            Lf = bank.lens[f]
            avail = min(max(Lf - beg, 0), n)
            if not (0 <= f < len(bank) and 0 <= beg and (beg < Lf or avail == 0)
                    and bank.offs[f] + beg + avail <= bank.data.numel()):
                raise ValueError("plan: segment file %d at %d does not fit its bank" % (f, beg))
            row[:] = (1, bank.offs[f] + beg, avail)

        for b, s in enumerate(samples):
            if "reverb" in s:
                conv_row(sec["rev"][b], self.ir, s["reverb"]["ir"], T, 1)
            if "overlap" in s:
                d = s["overlap"]
                if not 0 <= d["shift"] < T:
                    raise ValueError("plan: overlap shift %d outside [0, %d)" % (d["shift"], T))
                Ts = T - d["shift"]
                seg_row(sec["ovseg"][b], self.ov, d["file"], d["beg"], Ts)
                if "ir" in d:
                    conv_row(sec["ovrev"][b], self.ir, d["ir"], Ts, 1)
                sec["ovmix"][b] = (1, d["shift"], 0)
                dbl["ovsnr"][b] = 10 ** (d["snr"] / 10.)
            if "noise" in s:
                d = s["noise"]
                seg_row(sec["nseg"][b], self.noise, d["file"], d["beg"], T)
                sec["nmix"][b] = (1, 0, 1)
                dbl["nsnr"][b] = 10 ** (d["snr"] / 10.)
            if "clip" in s:
                sec["clip"][b] = 1
                dbl["cf"][b] = float(s["clip"]["cf"])
            if "bandrop" in s:
                conv_row(sec["bd"][b], self.bd, s["bandrop"]["filt"], T, 0)
            if "downsample" in s:
                conv_row(sec["ds"][b], self.ds, s["downsample"]["filt"], T, 0)
        return DistortionPlan(B, T, samples, table, offs)

    def sample_report(self, plan):
        """The reference's per-sample ``report`` dicts (later stages overwrite shared keys)."""
        out = []
        for s in plan.samples:
            r = {}
            if "reverb" in s:
                r["ir_file"] = self.ir.names[s["reverb"]["ir"]]
            if "overlap" in s:
                r["snr"] = s["overlap"]["snr"]
            if "noise" in s:
                r["snr"] = s["noise"]["snr"]
            if "clip" in s:
                r["clip_factor"] = s["clip"]["cf"]
            if "bandrop" in s:
                r["filt_file"] = self.bd.names[s["bandrop"]["filt"]]
            if "downsample" in s:
                r["filt_file"] = self.ds.names[s["downsample"]["filt"]]
            out.append(r)
        return out

    # ---- device stages -------------------------------------------------------------------
    def upload(self, plan, out=None):
        """Copy the plan table to the device (one H2D copy); into `out` when given (a graph
        replays with a newly uploaded plan this way)."""
        src = torch.from_numpy(plan.table)
        if self.device.type == "cuda":
            src = src.pin_memory()
        if out is None:
            return src.to(self.device, non_blocking=True)
        if out.numel() != src.numel() or out.dtype != torch.int64:
            raise ValueError("upload: table of %d int64 expected, got %d %s"
                             % (src.numel(), out.numel(), out.dtype))
        out.copy_(src, non_blocking=True)
        return out

    def _conv(self, x, bank, jobs, B, T, ldx):
        nbytes = ctypes.c_long(0)
        ops.call("pase_fft_conv_workspace", B, T, bank.lmax, ctypes.addressof(nbytes))
        ws = torch.empty((nbytes.value + 15) // 16 * 4, dtype=torch.float32, device=x.device)
        ops.call("pase_fft_conv", x, ldx, bank.data, bank.data.numel(), jobs, B, T, bank.lmax,
                 self.twiddle, ws, ws.numel() * 4, x, ldx)

    def run(self, y, table, offsets, overlap=None, d=1):
        """Apply every enabled stage in place to y ((B, T) contiguous fp32 on the device) with
        the device plan `table`; writes the (B, T/d) overlap label into `overlap` if given."""
        B, T = y.shape

        def sec(name):
            a, w = offsets[name]
            v = table[a:a + B * w]
            return v.view(torch.float64) if name in _DBL_SECTIONS else v

        names = [n for n, _ in self.stages]
        seg = torch.empty((B, T), dtype=torch.float32, device=y.device) \
            if ("overlap" in names or "noise" in names) else None
        for name in names:
            if name == "reverb":
                self._conv(y, self.ir, sec("rev"), B, T, T)
            elif name == "overlap":
                ops.call("pase_segment_gather", self.ov.data, self.ov.data.numel(), sec("ovseg"),
                         B, T, seg, T)
                if self.ov_reverb:
                    self._conv(seg, self.ir, sec("ovrev"), B, T, T)
                ops.call("pase_noise_mix", y, T, seg, T, sec("ovmix"), sec("ovsnr"), B, T)
            elif name == "noise":
                ops.call("pase_segment_gather", self.noise.data, self.noise.data.numel(),
                         sec("nseg"), B, T, seg, T)
                ops.call("pase_noise_mix", y, T, seg, T, sec("nmix"), sec("nsnr"), B, T)
            elif name == "clip":
                ops.call("pase_clip", y, T, sec("clip"), sec("cf"), B, T)
            elif name == "bandrop":
                self._conv(y, self.bd, sec("bd"), B, T, T)
            elif name == "downsample":
                self._conv(y, self.ds, sec("ds"), B, T, T)
        if overlap is not None:
            if "overlap" in names:
                ops.call("pase_overlap_label", sec("ovmix"), B, T, d, overlap, T // d)
            else:
                overlap.zero_()
        return y

    def apply(self, chunk, plan, overlap=None):
        """Distort a (B, 1, T) or (B, T) fp32 batch with `plan`.  Returns the distorted copy
        (same shape; `chunk` is not modified) and, when `overlap` ((B, 1, T/d) or (B, T/d))
        is given, the overlap label as a new tensor of its shape."""
        if chunk.dtype != torch.float32 or chunk.dim() not in (2, 3) or \
                (chunk.dim() == 3 and chunk.shape[1] != 1):
            raise ValueError("apply: chunk must be (B, 1, T) or (B, T) fp32, got %s %s"
                             % (tuple(chunk.shape), chunk.dtype))
        B, T = chunk.shape[0], chunk.shape[-1]
        if (B, T) != (plan.B, plan.T):
            raise ValueError("apply: plan is for B=%d T=%d, chunk is B=%d T=%d"
                             % (plan.B, plan.T, B, T))
        y = chunk.reshape(B, T).clone(memory_format=torch.contiguous_format)
        lab, d = None, 1
        if overlap is not None:
            n = overlap.shape[-1]
            if n <= 0 or T % n != 0 or overlap.numel() != B * n:
                raise ValueError("apply: overlap label length %d must divide T=%d" % (n, T))
            d = T // n
            lab = torch.empty((B, n), dtype=torch.float32, device=y.device)
        self.run(y, self.upload(plan), plan.offsets, lab, d)
        y = y.view(chunk.shape)
        return (y, None if lab is None else lab.view(overlap.shape))

    def __call__(self, batch):
        chunk = batch["chunk"]
        B, T = chunk.shape[0], chunk.shape[-1]
        plan = self.plan(B, T)
        y, lab = self.apply(chunk, plan, batch.get("overlap"))
        batch["chunk"] = y
        if lab is not None:
            batch["overlap"] = lab
        if self.report:
            return batch, self.sample_report(plan)
        return batch


_UNSUPPORTED = {
    "codec2": ("pycodec2 (Codec2 transcoding)", "codec2_p"),
    "chop": ("webrtcvad (the Chopper's voice activity detector)", "chop_p"),
    "speed": ("a SpeedChange port", "speed_p"),
    "resample": ("a Resample port", "resample_p"),
}


def config_distortions(reverb_irfiles=None, reverb_fmt='imp', reverb_data_root='.',
                       reverb_p=0.5, reverb_cache=False, overlap_dir=None, overlap_list=None,
                       overlap_snrs=[0, 5, 10], overlap_reverb=False, overlap_p=0.5,
                       noises_dir=None, noises_snrs=[0, 5, 10], noises_p=0.5,
                       noises_cache=False, speed_range=None, speed_p=0.5, resample_factors=[],
                       resample_p=0.5, bandrop_irfiles=[], bandrop_fmt='npy',
                       bandrop_data_root='.', bandrop_p=0.5, downsample_irfiles=[],
                       downsample_fmt='npy', downsample_data_root='.', downsample_p=0.5,
                       clip_factors=[], clip_p=0.5, chop_factors=[], max_chops=5, chop_p=0.5,
                       codec2_p=0.3, codec2_kbps=1600, codec2_cachedir=None, codec2_cache=False,
                       report=False, device="cuda"):
    """The reference's keyword signature (transforms.py:38-74) plus `device`.  Returns a
    :class:`Distortions`, or None when no stage is enabled.  Stages that need code this
    project lacks raise NotImplementedError naming the key to set to 0 (note the reference's
    default codec2_p=0.3 enables codec2)."""
    enabled = {
        "codec2": codec2_p > 0,
        "chop": chop_p > 0 and len(chop_factors) > 0,
        "speed": speed_p > 0 and speed_range is not None,
        "resample": resample_p > 0 and len(resample_factors) > 0,
    }
    for name, on in enabled.items():
        if on:
            dep, key = _UNSUPPORTED[name]
            raise NotImplementedError(
                "distortion stage '%s' needs %s, which this project does not have; set %s=0"
                % (name, dep, key))
    cfg = dict(locals())
    d = Distortions(cfg, device)
    return d if d.stages else None
