"""Deterministic synthetic data banks (IRs, FIRs, noise / overlap wavs) and the cases of the
distortion goldens (tests/golden/distortions.pt).  make_distortion_golden.py and the tests
rebuild the same files from these seeds, so no audio is committed.

Noise directories hold one wav each and overlap files come from a list file, so the file
order the reference's glob sees does not depend on the filesystem.
"""
import os

import numpy as np
import torch

IR_LENS = (24000, 7000, 4097)
FIR_LENS = (101, 103, 100)
DS_LENS = (101,)
OV_LENS = (3000, 40000)              # shorter than any T - s at T = 16000, and longer than T
NOISE_LENS = (9000, 16000, 50000)    # shorter than, equal to and longer than T = 16000


def make_ir(L, seed):
    rng = np.random.RandomState(seed)
    t = np.arange(L)
    h = rng.randn(L) * np.exp(-t / (L / 6.0)) * 0.3
    pk = min(40 + seed % 17, L - 1)
    h[pk] = 1.5 + rng.rand()
    return h


def make_fir(L, seed):
    rng = np.random.RandomState(seed)
    n = np.arange(L) - (L - 1) / 2.0
    fc = 0.15 + 0.2 * rng.rand()
    h = 2 * fc * np.sinc(2 * fc * n) * np.hamming(L)
    return h + 1e-3 * rng.randn(L)


def make_wav(n, seed):
    rng = np.random.RandomState(seed)
    env = 0.5 + 0.5 * np.sin(np.linspace(0, 7.0 + seed % 5, n)) ** 2
    return np.clip(rng.randn(n) * 4000 * env, -32768, 32767).astype(np.int16)


def make_chunk(B, T, seed):
    rng = np.random.RandomState(seed)
    t = np.arange(T)
    env = 0.2 + np.abs(np.sin(2 * np.pi * t / 4000.0))[None, :]
    x = rng.randn(B, T) * env * 0.1 + 0.05 * np.sin(2 * np.pi * 220 * t / 16000.0)[None, :]
    return x.astype(np.float32)


def build_banks(root):
    """Writes every bank under `root`; returns the paths config_distortions needs."""
    from scipy.io import wavfile
    p = {k: os.path.join(root, k) for k in ("irs", "firs", "ds", "ov")}
    for d in p.values():
        os.makedirs(d, exist_ok=True)
    p["ir_files"] = []
    for i, L in enumerate(IR_LENS):
        name = "ir_%d.npy" % L
        np.save(os.path.join(p["irs"], name), make_ir(L, 100 + i))
        p["ir_files"].append(name)
    p["fir_files"] = []
    for i, L in enumerate(FIR_LENS):
        name = "fir_%d.npy" % L
        np.save(os.path.join(p["firs"], name), make_fir(L, 200 + i))
        p["fir_files"].append(name)
    p["ds_files"] = []
    for i, L in enumerate(DS_LENS):
        name = "ds_%d.npy" % L
        np.save(os.path.join(p["ds"], name), make_fir(L, 300 + i))
        p["ds_files"].append(name)
    names = []
    for i, n in enumerate(OV_LENS):
        name = "ov_%d.wav" % n
        wavfile.write(os.path.join(p["ov"], name), 16000, make_wav(n, 400 + i))
        names.append(name)
    p["ov_list"] = os.path.join(root, "ov.scp")
    with open(p["ov_list"], "w") as fh:
        fh.write("\n".join(names) + "\n")
    p["noise_dirs"] = []
    for i, n in enumerate(NOISE_LENS):
        d = os.path.join(root, "noise%d" % i)
        os.makedirs(d, exist_ok=True)
        wavfile.write(os.path.join(d, "n_%d.wav" % n), 16000, make_wav(n, 500 + i))
        p["noise_dirs"].append(d)
    return p


def raw_banks(paths):
    """float64 arrays as the reference reads them (PCM16 / 32768), for the float64 oracle."""
    from scipy.io import wavfile

    def wav(f):
        return wavfile.read(f)[1].astype(np.float64) / 32768.0
    return {
        "irs": [np.load(os.path.join(paths["irs"], f)) for f in paths["ir_files"]],
        "bandrop": [np.load(os.path.join(paths["firs"], f)) for f in paths["fir_files"]],
        "downsample": [np.load(os.path.join(paths["ds"], f)) for f in paths["ds_files"]],
        "overlap": [wav(os.path.join(paths["ov"], n)) for n in
                    open(paths["ov_list"]).read().split()],
        "noise": [wav(os.path.join(d, os.listdir(d)[0])) for d in paths["noise_dirs"]],
    }


def base_cfg(paths):
    """Every stage off (codec2 and chop too); IR / filter lists explicit."""
    return dict(reverb_irfiles=list(paths["ir_files"]), reverb_fmt="npy",
                reverb_data_root=paths["irs"], reverb_p=0.0,
                overlap_dir=paths["ov"], overlap_list=paths["ov_list"], overlap_snrs=[5, 7.5, 10],
                overlap_reverb=False, overlap_p=0.0,
                noises_dir=list(paths["noise_dirs"]), noises_snrs=[0, 5, 10], noises_p=0.0,
                clip_factors=[0.1, 0.3, 0.5], clip_p=0.0,
                bandrop_irfiles=list(paths["fir_files"]), bandrop_fmt="npy",
                bandrop_data_root=paths["firs"], bandrop_p=0.0,
                downsample_irfiles=list(paths["ds_files"]), downsample_fmt="npy",
                downsample_data_root=paths["ds"], downsample_p=0.0,
                chop_p=0.0, codec2_p=0.0)


PASE_PLUS_P = dict(reverb_p=0.5, overlap_p=0.1, overlap_reverb=True, noises_p=0.4, clip_p=0.2,
                   bandrop_p=0.35, downsample_p=0.25)

# name -> (overrides, B, T, d, seed)
CASES = {
    "reverb_24000": (dict(reverb_p=1.0, reverb_irfiles=["ir_24000.npy"]), 2, 16000, 160, 11),
    "reverb_7000": (dict(reverb_p=1.0, reverb_irfiles=["ir_7000.npy"]), 2, 16000, 160, 12),
    "reverb_4097": (dict(reverb_p=1.0, reverb_irfiles=["ir_4097.npy"]), 2, 16000, 160, 13),
    "overlap": (dict(overlap_p=1.0), 8, 16000, 160, 14),
    "overlap_reverb": (dict(overlap_p=1.0, overlap_reverb=True), 8, 16000, 160, 15),
    "noise": (dict(noises_p=1.0), 8, 16000, 160, 16),
    "clip": (dict(clip_p=1.0), 4, 16000, 160, 17),
    "bandrop": (dict(bandrop_p=1.0), 6, 16000, 160, 18),
    "downsample": (dict(downsample_p=1.0), 2, 16000, 160, 19),
    "pase_plus": (dict(PASE_PLUS_P), 32, 16000, 160, 20),
    "all_48000": (dict(reverb_p=1.0, overlap_p=1.0, overlap_reverb=True, noises_p=1.0,
                       clip_p=1.0, bandrop_p=1.0, downsample_p=1.0), 3, 48000, 160, 21),
}


# What the golden keeps of each (B, T) reference output: every sample of FULL_CASES; for every
# case the first and last EDGE samples of each row (the shifted / padded ends), every
# STRIDE-th sample (a prime stride, so the samples walk across the 4096-sample blocks), the
# row's L2 norm and max |y|.
FULL_CASES = ("reverb_24000",)
EDGE = 256
STRIDE = 97


def golden_view(y):
    """(B, T) tensor -> the parts of it the golden keeps, concatenated per row."""
    return torch.cat([y[:, :EDGE], y[:, -EDGE:], y[:, ::STRIDE]], dim=1).contiguous()


def case_cfg(name, paths):
    over, B, T, d, seed = CASES[name]
    cfg = base_cfg(paths)
    cfg.update(over)
    return cfg, B, T, d, seed
