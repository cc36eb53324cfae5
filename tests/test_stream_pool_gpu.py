"""WaveFe.streams() / StreamPool on the GPU: bit-equal to the whole-recording forward in every
precision with CPU and CUDA blocks mixed (a stream of at most 512 frames, where that forward
runs the parallel QRNN scan: bit-equal to the recording pushed whole, close to the forward), 256
streams of 10 ms pushes against extract_long,
rounds split into several packs, launches per round independent of the number of streams, two
host-to-device copies and no device-to-host copy per round, and one allocation per round after
warm-up."""
import random

import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode

import pase_b200.ops as ops
from pase_b200 import encoder as enc
from helpers import resolve_cfg, fill_state_dict, seeded_randn, assert_close
from pase_b200.frontend import WaveFe

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tf32", "3xtf32", "3xf16", "bf16"]
CFGS = ["cfg/frontend/PASE.cfg", "cfg/frontend/PASE+.cfg"]
SEED = 11
W = 81920


def _model(cfg_name, precision="3xf16"):
    m = WaveFe(**resolve_cfg(cfg_name))
    m.load_state_dict(fill_state_dict(m.state_dict(), SEED))
    m.precision = precision
    return m.cuda().eval()


def _windowable(L):
    """L moved off the lengths whose dense skips no window reproduces (PASE+: mod 160 in
    151..159, encoder.check_windowable)."""
    return L - 10 if L % 160 >= 151 else L


def _schedule(rng, lengths, starts):
    """Per call ({k: (a, b)}, [k finishing]): stream k opens at call starts[k], sends blocks of
    1..30000 samples (one of 90000 first for k % 5 == 1, past the window chunk) and finishes
    with its last block (even k) or one call later (odd k)."""
    pos, done, calls, c = [0] * len(lengths), [False] * len(lengths), [], 0
    while not all(done):
        blocks, fin = {}, []
        for k, L in enumerate(lengths):
            if c < starts[k] or done[k]:
                continue
            if pos[k] < L:
                n = 90000 if (k % 5 == 1 and pos[k] == 0) else rng.randint(1, 30000)
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


def _run_pool(pool, xs, calls, starts, on_gpu):
    ids, outs = {}, {k: [] for k in range(len(xs))}
    for c, (blocks, fin) in enumerate(calls):
        for k, s in enumerate(starts):
            if s == c:
                ids[k] = pool.open()
        res = pool.push({ids[k]: (xs[k][a:b].cuda() if on_gpu(k, c) else xs[k][a:b])
                         for k, (a, b) in blocks.items()}, [ids[k] for k in fin])
        for k in set(blocks) | set(fin):
            y = res[ids[k]]
            assert y.is_cuda and y.dim() == 3 and y.shape[0] == 1
            outs[k].append(y)
    return {k: torch.cat(v, 2) for k, v in outs.items()}


def _reference(m, x):
    """The frames a stream of x gives: those of the whole-recording forward above 512 frames.
    At most 512 frames that forward runs the parallel QRNN scan, so the reference is x pushed
    whole into a one-stream pool, checked close to the forward."""
    with torch.no_grad():
        y = m(x.view(1, 1, -1).cuda())
    if y.shape[2] > enc.MIN_WINDOW_FRAMES:
        return y
    pool = m.streams(1)
    i = pool.open()
    got = pool.push({i: x}, finish=[i])[i]
    tol = (1e-2, 1e-3) if m.resolved_precision() in ("tf32", "bf16") else (1e-4, 1e-5)
    assert_close(got, y, *tol, "%d samples pushed whole" % x.numel())
    return got


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("cfg_name", CFGS)
def test_pool_bit_equal_to_feature_streams(cfg_name, precision):
    m = _model(cfg_name, precision)
    rng = random.Random(cfg_name + precision)
    lengths = [_windowable(rng.randrange(26000, 200000)) for _ in range(16)]
    lengths[3] = 40000                                         # < 512 frames
    starts = [k // 3 for k in range(16)]
    xs = [seeded_randn((L,), 200 + k, 0.5) for k, L in enumerate(lengths)]
    calls = _schedule(rng, lengths, starts)
    got = _run_pool(m.streams(16), xs, calls, starts, lambda k, c: (k + c) % 2 == 0)
    for k in range(16):
        ref = _reference(m, xs[k])
        assert got[k].shape == ref.shape
        assert torch.equal(got[k], ref), (k, float((got[k] - ref).abs().max()))


def test_256_streams_of_10ms_pushes_equal_extract_long():
    m = _model("cfg/frontend/PASE+.cfg", "bf16")
    N, L, hop = 256, 160000, 160
    xs = torch.randn(N, L, generator=torch.Generator().manual_seed(3)) * 0.5
    pool = m.streams(N)
    ids = [pool.open() for _ in range(N)]
    outs = [[] for _ in range(N)]
    for a in range(0, L, hop):
        res = pool.push({i: xs[k, a:a + hop] for k, i in enumerate(ids)})
        for k, i in enumerate(ids):
            outs[k].append(res[i])
    res = pool.push({}, finish=ids)
    for k, i in enumerate(ids):
        got = torch.cat(outs[k] + [res[i]], 2)
        ref = m.extract_long(xs[k])
        assert got.shape == ref.shape and torch.equal(got, ref), k
    assert len(pool) == 0


def test_round_split_into_packs():
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    rng = random.Random(9)
    lengths = [_windowable(rng.randrange(90000, 160000)) for _ in range(12)]
    xs = [seeded_randn((L,), 300 + k, 0.5) for k, L in enumerate(lengths)]
    starts = [0] * 12
    calls = _schedule(rng, lengths, starts)
    n0 = ops.launch_count
    got = _run_pool(m.streams(12, max_samples=60000), xs, calls, starts, lambda k, c: k % 3 == 0)
    packed = ops.launch_count - n0
    n0 = ops.launch_count
    one = _run_pool(m.streams(12, max_samples=1 << 22), xs, calls, starts, lambda k, c: False)
    assert packed > ops.launch_count - n0                      # more packs, more launches
    for k in range(12):
        ref = _reference(m, xs[k])
        assert torch.equal(got[k], ref) and torch.equal(one[k], ref), k


def _warm_pool(m, N, hop=160, rounds=200):
    """A pool of N streams past their first tail (every round runs one segment per stream)."""
    pool = m.streams(N, max_samples=1 << 21)
    ids = [pool.open() for _ in range(N)]
    xs = torch.randn(N, hop * (rounds + 40), generator=torch.Generator().manual_seed(N)) * 0.5
    for r in range(rounds):
        pool.push({i: xs[k, r * hop:(r + 1) * hop] for k, i in enumerate(ids)})
    torch.cuda.synchronize()
    return pool, ids, xs, rounds * hop


class _Copies(TorchDispatchMode):
    """Counts the host-to-device and device-to-host copies issued from Python inside the block.
    (Counted at the dispatcher rather than with torch.profiler: a profiler session opened after
    earlier sessions in the same process can miss copies, so this test opens none.)"""

    def __init__(self):
        super().__init__()
        self.h2d = self.d2h = 0

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        out = func(*args, **kwargs)
        if func is torch.ops.aten.copy_.default:
            dst, src = args[0], args[1]
            self.h2d += int(dst.is_cuda and not src.is_cuda)
            self.d2h += int(src.is_cuda and not dst.is_cuda)
        elif func is torch.ops.aten._to_copy.default:
            src = args[0]
            self.h2d += int(out.is_cuda and not src.is_cuda)
            self.d2h += int(src.is_cuda and not out.is_cuda)
        elif func is torch.ops.aten._local_scalar_dense.default and args[0].is_cuda:
            self.d2h += 1                                   # .item() / .tolist() of a CUDA tensor
        return out


def test_launches_copies_and_allocations_per_round():
    m = _model("cfg/frontend/PASE+.cfg", "3xf16")
    launches = {}
    for N in (1, 64):
        pool, ids, xs, a = _warm_pool(m, N)
        n0 = ops.launch_count
        res = pool.push({i: xs[k, a:a + 160] for k, i in enumerate(ids)})
        launches[N] = ops.launch_count - n0
        assert all(res[i].shape[2] == 1 for i in ids)
        a += 160
        # after warm-up a round allocates its output only
        torch.cuda.synchronize()
        c0 = torch.cuda.memory_stats()["allocation.all.allocated"]
        pool.push({i: xs[k, a:a + 160] for k, i in enumerate(ids)})
        torch.cuda.synchronize()
        assert torch.cuda.memory_stats()["allocation.all.allocated"] - c0 == 1, N
        a += 160
        with _Copies() as c:
            pool.push({i: xs[k, a:a + 160] for k, i in enumerate(ids)})
            torch.cuda.synchronize()
        assert (c.h2d, c.d2h) == (2, 0), (N, c.h2d, c.d2h)
    assert launches[1] == launches[64] > 0, launches


def test_refusals_on_the_device():
    m = _model("cfg/frontend/PASE+.cfg")
    pool = m.streams(2)
    a = pool.open()
    pool.push({a: torch.zeros(30000).cuda()})
    n0 = ops.launch_count
    with pytest.raises(ValueError, match="mode"):
        m.streams(2, mode="avg_norm")
    with pytest.raises(ValueError, match="window"):
        m.streams(2, window=1000)
    with pytest.raises(ValueError, match="shorter"):
        b = pool.open()
        pool.push({a: torch.zeros(160).cuda(), b: torch.zeros(100)}, finish=[b])
    with pytest.raises(NotImplementedError):
        pool.push({a: torch.zeros(1679).cuda()}, finish=[a])
    with pytest.raises(RuntimeError, match="max_streams"):
        pool.open()
    m.train()
    with pytest.raises(RuntimeError, match="eval"):
        pool.push({a: torch.zeros(10)})
    m.eval()
    m.cpu()
    with pytest.raises(RuntimeError, match="CUDA"):
        pool.push({a: torch.zeros(10)})
    assert ops.launch_count == n0
    assert pool._streams[a].n == 30000 and enc.final_frames(m.cfg, 30000) == \
        pool._streams[a].done
