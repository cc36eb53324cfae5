"""Generates tests/golden/distortions.pt from the UNMODIFIED reference distortions
(pase/transforms.py config_distortions / PCompose).  Run:
    PASE_REFERENCE_ROOT=<checkout of santi-pdp/pase> python tests/golden/make_distortion_golden.py

pase.transforms imports feature-extraction packages the distortions never use; they get
import-only stubs here, and soundfile gets a `read` built on scipy's wav reader (PCM16 / 32768,
the values soundfile returns).  The banks come from the seeds in distortion_banks.py.  For every
case the global `random` / `np.random` are seeded once, the reference PCompose runs on samples
0..B-1 in turn, and each sample's draw stream (random.random, random.choice,
np.random.randint) is recorded alongside its overlap label and its float32 output.  Outputs
are kept in full for distortion_banks.FULL_CASES; for every case the golden keeps
golden_view (both row edges and a strided sample), the row norms and max |y|.
"""
import json
import os
import random
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from distortion_banks import (CASES, FULL_CASES, build_banks, case_cfg, golden_view,  # noqa: E402
                              make_chunk)

REF_ROOT = os.environ.get("PASE_REFERENCE_ROOT", "")


def install_stubs():
    from scipy.io import wavfile

    def stub(name, **attrs):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    def unavailable(*a, **k):
        raise RuntimeError("import-only stub")

    stub("gammatone")
    stub("gammatone.gtgram", gtgram=unavailable)
    stub("pysptk")
    stub("python_speech_features", logfbank=unavailable)
    stub("librosa")
    stub("ahoproc_tools")
    stub("ahoproc_tools.interpolate", interpolation=unavailable)
    stub("ahoproc_tools.io")

    def sf_read(path):
        rate, data = wavfile.read(path)
        assert data.dtype == np.int16, data.dtype
        return data.astype(np.float64) / 32768.0, rate
    stub("soundfile", read=sf_read)


class Recorder:
    """Wraps random.random, random.choice and np.random.randint; logs every draw."""

    def __init__(self):
        self.log = []

    def __enter__(self):
        self._saved = (random.random, random.choice, np.random.randint)
        r0, c0, i0 = self._saved

        def rnd():
            v = r0()
            self.log.append(["random", v])
            return v

        def choice(seq):
            v = c0(seq)
            self.log.append(["choice", len(seq), v])
            return v

        def randint(low, high=None, *a, **k):
            v = i0(low, high, *a, **k)
            self.log.append(["randint", int(low), int(high), int(v)])
            return v
        random.random, random.choice, np.random.randint = rnd, choice, randint
        return self

    def __exit__(self, *exc):
        random.random, random.choice, np.random.randint = self._saved


def main():
    if not os.path.isdir(os.path.join(REF_ROOT, "pase")):
        raise SystemExit("set PASE_REFERENCE_ROOT to a checkout of santi-pdp/pase")
    install_stubs()
    sys.path.insert(0, REF_ROOT)
    import pase.transforms as RT
    out = {}
    with tempfile.TemporaryDirectory() as root:
        paths = build_banks(root)
        for name in CASES:
            cfg, B, T, d, seed = case_cfg(name, paths)
            comp = RT.config_distortions(report=True, **cfg)
            x = make_chunk(B, T, seed)
            random.seed(seed)
            np.random.seed(seed)
            ys, labs, streams, reports = [], [], [], []
            for b in range(B):
                pkg = {"chunk": torch.from_numpy(x[b].copy()),
                       "overlap": torch.zeros(T // d), "dec_resolution": d}
                with Recorder() as rec:
                    pkg, rep = comp(pkg)
                ys.append(pkg["chunk"].float().reshape(-1))
                labs.append(pkg["overlap"].float().reshape(-1))
                streams.append(rec.log)
                reports.append({k: v for k, v in rep.items()})
            Y = torch.stack(ys)
            out[name + "/y_view"] = golden_view(Y)
            out[name + "/y_norm"] = Y.double().norm(dim=1)
            out[name + "/y_amax"] = Y.abs().amax(dim=1)
            if name in FULL_CASES:
                out[name + "/y"] = Y
            out[name + "/overlap"] = torch.stack(labs)
            out[name + "/meta"] = json.dumps({"B": B, "T": T, "d": d, "seed": seed,
                                              "streams": streams, "reports": reports})
            print("%-16s B=%d T=%d  draws/sample %.1f" % (name, B, T,
                                                          np.mean([len(s) for s in streams])))
    torch.save(out, os.path.join(HERE, "distortions.pt"))


if __name__ == "__main__":
    main()
