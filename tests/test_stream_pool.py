"""Host side of WaveFe.streams() / StreamPool on CPU, every kernel launch replaced by its torch
emulation (tests/emul/): many staggered streams against one one-stream pool each fed
the same blocks, against the recording pushed whole and against the B=1 forward, slot reuse, a
finish folded into the last block, the pack bound, and refusals raised before any launch with no
stream changed.  The emulated GEMMs round differently for different segment lengths, so here a
stream equals another bit for bit only when both are cut into the same segments; that the frames
do not depend on the cuts is checked on the GPU (tests/test_stream_pool_gpu.py)."""
import random

import pytest
import torch

import emul
from helpers import resolve_cfg, fill_state_dict, seeded_randn, assert_close
import pase_b200.ops as ops
from pase_b200 import encoder as enc
from pase_b200.frontend import StreamPool, WaveFe
from test_extract_long import single

CFGS = ["cfg/frontend/PASE.cfg", "cfg/frontend/PASE+.cfg"]
CPU = torch.device("cpu")
W = 81920


@pytest.fixture()
def gathers(monkeypatch):
    """Emulated launches; records every pase_stream_gather table, and every launch's name in
    gathers.names."""
    seen = _Seen()

    def call(name, *args):
        seen.names.append(name)
        if name == "pase_stream_gather":
            seen.append(args[4][:8 * args[5]].view(-1, 8).clone())
        return emul.call(name, *args)
    monkeypatch.setattr(ops, "call", call)
    yield seen


class _Seen(list):
    def __init__(self):
        super().__init__()
        self.names = []


def make_model(cfg_name, precision="fp32", seed=11):
    model = WaveFe(**resolve_cfg(cfg_name))
    model.precision = precision
    model.load_state_dict(fill_state_dict(model.state_dict(), seed))
    return model.eval()


def schedule(rng, lengths, starts, big=()):
    """Calls of a pool: per call ({k: (a, b)} blocks, [k finishing]).  Stream k opens at call
    starts[k], sends blocks of 1..30000 samples (its first one of 90000 when k in big) and
    finishes with its last block (even k) or in the call after it (odd k)."""
    pos, done, calls, c = [0] * len(lengths), [False] * len(lengths), [], 0
    while not all(done):
        blocks, fin = {}, []
        for k, L in enumerate(lengths):
            if c < starts[k] or done[k]:
                continue
            if pos[k] < L:
                n = 90000 if (k in big and pos[k] == 0) else rng.randint(1, 30000)
                blocks[k] = (pos[k], min(L, pos[k] + n))
                pos[k] = blocks[k][1]
                if pos[k] == L and k % 2 == 0:
                    fin.append(k)
                    done[k] = True
            else:
                fin.append(k)
                done[k] = True
        calls.append((blocks, fin))
        c += 1
    return calls


def run_pool(pool, xs, calls, starts):
    ids, outs = {}, {k: [] for k in range(len(xs))}
    for c, (blocks, fin) in enumerate(calls):
        for k, s in enumerate(starts):
            if s == c:
                ids[k] = pool.open()
        res = pool.push({ids[k]: xs[k][a:b] for k, (a, b) in blocks.items()},
                        [ids[k] for k in fin])
        assert set(res) == {ids[k] for k in set(blocks) | set(fin)}
        for k in set(blocks) | set(fin):
            outs[k].append(res[ids[k]])
    return {k: torch.cat(v, 2) for k, v in outs.items()}


def alone(model, x, calls):
    """x fed to a fresh one-stream pool in the blocks and finishes of `calls` ({None: (a, b)}
    blocks, [None] finishing), or whole in one push that also finishes it (calls None)."""
    pool = StreamPool(model, CPU, 1, W)
    i = pool.open()
    if calls is None:
        return pool.push({i: x}, finish=[i])[i]
    return torch.cat([pool.push({i: x[a:b] for a, b in blocks.values()}, [i] if fin else [])[i]
                      for blocks, fin in calls], 2)


def calls_of(calls, k):
    return [({k: c[0][k]} if k in c[0] else {}, [k] if k in c[1] else [])
            for c in calls if k in c[0] or k in c[1]]


@pytest.mark.parametrize("cfg_name", CFGS)
def test_pool_matches_one_stream_pools(cfg_name, gathers):
    model = make_model(cfg_name)
    lengths = [50000, 100000, 30000, 70000, 120000, 26000]      # 0: < 512 frames
    starts = [0, 0, 1, 2, 2, 4]
    xs = [seeded_randn((L,), 100 + k, 0.5) for k, L in enumerate(lengths)]
    calls = schedule(random.Random(5), lengths, starts, big=(1,))   # a block past the chunk
    assert max(b - a for blocks, _ in calls for a, b in blocks.values()) > W
    max_samples = 60000
    pool = StreamPool(model, CPU, 6, W, max_samples)
    got = run_pool(pool, xs, calls, starts)
    assert len(pool) == 0
    for k in range(len(xs)):
        ref = alone(model, xs[k], calls_of(calls, k))
        assert got[k].shape == ref.shape == (1, model.emb_dim,
                                             enc.frame_counts(model.cfg, lengths[k])[-1])
        assert torch.equal(got[k], ref), (k, float((got[k] - ref).abs().max()))
        assert_close(got[k], alone(model, xs[k], None), 1e-5, 1e-6, "stream %d" % k)
        assert_close(got[k], single(model, xs[k]), 1e-4, 1e-5, "stream %d" % k)
    # every pack within max_samples (a longer segment alone), no slot twice in one pack
    assert gathers
    for t in gathers:
        segs = t[t[:, 6] > 0]
        assert int(segs[:, 6].sum()) <= max_samples or len(segs) == 1
        assert len(set(t[:, 0].tolist())) == len(t)


def test_reused_slot_equals_fresh_stream(gathers):
    model = make_model("cfg/frontend/PASE+.cfg")
    pool = StreamPool(model, CPU, 2, W)
    x, y = seeded_randn((60000,), 1, 0.5), seeded_randn((40000,), 2, 0.5)
    a, b = pool.open(), pool.open()
    pool.push({a: x[:30000], b: y[:30000]})
    pool.push({a: x[30000:]}, finish=[a])                   # a's slot is free again
    c = pool.open()
    assert pool._streams[c].slot == 0
    outs = [pool.push({c: y[:25000], b: y[30000:]})[c], pool.push({c: y[25000:]}, [b, c])[c]]
    ref = alone(model, y, [({0: (0, 25000)}, []), ({0: (25000, 40000)}, []), ({}, [0])])
    assert torch.equal(torch.cat(outs, 2), ref)


def test_finish_with_last_block_runs_one_segment(gathers):
    model = make_model("cfg/frontend/PASE+.cfg")
    L = W + 160 * 30 + 77
    x = seeded_randn((L,), 21, 0.5)
    alone(model, x, None)
    segs = [int((t[:, 6] > 0).sum()) for t in gathers]
    assert segs == [1] * len(enc.plan_windows(model.cfg, L, W)) == [1, 1]
    pool = StreamPool(model, CPU, 1, W)
    i = pool.open()
    del gathers[:]
    pool.push({i: x[:50000]})
    pool.push({i: x[50000:]}, finish=[i])             # one piece, planned at the end
    assert [int((t[:, 6] > 0).sum()) for t in gathers] == [1, 1]


def _counters(pool):
    return {i: (s.slot, s.n, s.done, s.keep) for i, s in pool._streams.items()}


def test_refusals_before_any_launch(gathers):
    model = make_model("cfg/frontend/PASE+.cfg", "3xf16")
    pool = StreamPool(model, CPU, 3, W)
    a, b, c = pool.open(), pool.open(), pool.open()
    pool.push({a: seeded_randn((30000,), 3, 0.5), b: torch.zeros(300), c: torch.zeros(100)})
    before, n0 = _counters(pool), len(gathers.names)
    bad = [
        (RuntimeError, "max_streams", lambda: pool.open()),
        (KeyError, "unknown", lambda: pool.push({a: torch.zeros(10), 99: torch.zeros(10)})),
        (ValueError, "shorter", lambda: pool.push({a: torch.zeros(10)}, finish=[b])),
        # 30000 + 1679 samples: L mod 160 = 159, no hop-aligned window pools it right
        (NotImplementedError, "pools its dense skips",
         lambda: pool.push({a: torch.zeros(1679)}, finish=[a])),
        (TypeError, "fp32", lambda: pool.push({a: torch.zeros(10, dtype=torch.float64)})),
        (ValueError, "recording", lambda: pool.push({a: torch.zeros(2, 10)})),
        (TypeError, "map", lambda: pool.push([torch.zeros(10)])),
    ]
    for exc, msg, fn in bad:
        with pytest.raises(exc, match=msg):
            fn()
        assert len(gathers.names) == n0 and _counters(pool) == before, msg
    model.train()
    with pytest.raises(RuntimeError, match="eval"):
        pool.push({a: torch.zeros(10)})
    with pytest.raises(RuntimeError, match="eval"):
        model.streams(4)
    model.eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        model.streams(4)
    with pytest.raises(ValueError, match="window"):
        StreamPool(model, CPU, 4, W - 160)
    assert len(gathers.names) == n0 and _counters(pool) == before
    pool.push({}, finish=[a])                               # a finished: its id is gone
    with pytest.raises(KeyError, match="finished"):
        pool.push({a: torch.zeros(10)})
