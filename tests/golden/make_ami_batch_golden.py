"""Generates tests/golden/ami_batch.pt from the UNMODIFIED reference data pipeline
(pase/dataset.py AmiSegTupleWavDataset + DictCollater, pase/transforms.py CachedCompose +
MIChunkWav / SingleChunkWav, and config_distortions for the distorted case).
Run:
    PASE_REFERENCE_ROOT=<checkout of santi-pdp/pase> python tests/golden/make_ami_batch_golden.py

The stubs of make_batch_golden.py.  For each case the paired corpus of ami_corpus.py is built,
the global random / np.random / torch generators are seeded once, and the dataset's
__getitem__ runs on each index of each batch in turn (what a num_workers=0 DataLoader does),
then DictCollater collates.  Kept per case: the utterances the dataset kept, every draw of every
sample (random.random, random.choice, np.random.randint, torch.rand), the parsed per-sample
choices, and per batch the shape and SHA-256 (batch_corpus.digest) of every clean collated
array, the first values of each, and for the distorted case the distorted chunk itself.
"""
import json
import os
import random
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ami_corpus import CASES, HOP, KEYS, SPLIT, T, build_ami_corpus, digest  # noqa: E402
from distortion_banks import build_banks, case_cfg  # noqa: E402
from make_batch_golden import VIEW, BatchRecorder, install_torchaudio_stub  # noqa: E402
from make_distortion_golden import install_stubs  # noqa: E402

REF_ROOT = os.environ.get("PASE_REFERENCE_ROOT", "")


def parse(index, log, n, paired, chunk_beg):
    """Per-sample choices from the draw log of one __getitem__: the neighbour (its index in
    the kept list), the random utterance, the channel, the window starts drawn, the scales."""
    k, ctxt = 0, index
    if log[0][0] == "choice" and isinstance(log[0][2], (list, tuple)):
        ctxt, k = int(log[0][2][0]), 1
    assert log[k][0] == "choice" and log[k][1] == n - 1
    rand = int(log[k][2])
    k += 1
    channel = None
    if paired:
        assert log[k][0] == "choice" and isinstance(log[k][2], str)
        channel = log[k][2]
        k += 1
    randints = []
    while k < len(log) and log[k][0] == "randint":
        randints.append(log[k][3])
        k += 1
    scale = []
    while k < len(log) and log[k][0] == "rand":
        scale.append(log[k][1])
        k += 1
    return {"index": index, "ctxt": ctxt, "rand": rand, "channel": channel,
            "chunk_beg": int(chunk_beg), "randints": randints, "scale": scale or None,
            "dist_log": log[k:]}


def main():
    if not os.path.isdir(os.path.join(REF_ROOT, "pase")):
        raise SystemExit("set PASE_REFERENCE_ROOT to a checkout of santi-pdp/pase")
    install_stubs()
    install_torchaudio_stub()
    sys.path.insert(0, REF_ROOT)
    import pase.transforms as RT
    from pase.dataset import AmiSegTupleWavDataset, DictCollater
    out = {}
    with tempfile.TemporaryDirectory() as root:
        data_root, cfg_path, cache = build_ami_corpus(root)
        bank_paths = build_banks(os.path.join(root, "banks"))
        for name, c in CASES.items():
            chunker = (RT.MIChunkWav if c["mi"] else RT.SingleChunkWav)(
                T, random_scale=c["random_scale"])
            trans, keys = [RT.ToTensor(), chunker], ["totensor", "chunk"]
            if c["cached"]:
                trans += [RT.FBanks(hop=HOP, name="fbank"), RT.MFCC(hop=HOP, name="mfcc")]
                keys += list(KEYS)
            dist = None
            if c["distortions"]:
                dist = RT.config_distortions(**case_cfg("pase_plus", bank_paths)[0])
            ds = AmiSegTupleWavDataset(
                data_root, cfg_path, SPLIT, transform=RT.CachedCompose(trans, keys, cache),
                distortion_transforms=dist, zero_speech_p=0, ihm2sdm=c["ihm2sdm"])
            coll = DictCollater()
            random.seed(c["seed"])
            np.random.seed(c["seed"])
            torch.manual_seed(c["seed"])
            meta = {"names": [w["filename"] for w in ds.wavs], "samples": [], "logs": [],
                    "arrays": []}
            for bi, idx in enumerate(c["batches"]):
                pkgs = []
                for i in idx:
                    with BatchRecorder() as rec:
                        pkgs.append(ds[i])
                    log = json.loads(json.dumps(rec.log))
                    meta["logs"].append(log)
                    meta["samples"].append(parse(i, log, len(ds.wavs), c["ihm2sdm"] is not None,
                                                 pkgs[-1]["chunk_beg_i"]))
                batch = coll(pkgs)
                arr = {}
                for k, v in batch.items():
                    a = v.float().numpy()
                    if c["distortions"] and k == "chunk":
                        out["%s/%d/chunk" % (name, bi)] = v.float().clone()
                        continue
                    arr[k] = {"shape": list(a.shape), "sha256": digest(a),
                              "view": [float(x) for x in a.reshape(a.shape[0], -1)[0, :VIEW]]}
                meta["arrays"].append(arr)
            out[name + "/meta"] = json.dumps(meta)
            print("%-22s %d utterances %s" % (name, len(ds.wavs),
                                             {k: v["shape"] for k, v in meta["arrays"][0].items()}))
    torch.save(out, os.path.join(HERE, "ami_batch.pt"))


if __name__ == "__main__":
    main()
