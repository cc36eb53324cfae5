"""The data-parallel GraphedTrainStep's refusals, on two CPU ranks (gloo): a peer_dp engine
without a process group, and a peer_dp engine built over another group than the step's.  The
engines are built over one-rank subgroups, which need no peer mapping and no GPU."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_train_step import _cpu_batcher, build_corpus, make_model


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, corpus, out):
    import pytest
    from pase_b200.graph import GraphedTrainStep
    from pase_b200.optim import FlatAdam
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        subs = [dist.new_group([q]) for q in range(world)]
        model = make_model("pase").train()
        batcher = _cpu_batcher(corpus, "pase", 8000)
        peer = FlatAdam(list(model.parameters()), lr=1e-3, peer_dp=True,
                        group=subs[rank]).bind_encoder(model.frontend)
        assert peer._peer is None                   # one rank: nothing to map
        with pytest.raises(NotImplementedError, match="peer_dp"):
            GraphedTrainStep(model, peer, batcher, 4)
        with pytest.raises(ValueError, match="another process group"):
            GraphedTrainStep(model, peer, batcher, 4, group=dist.group.WORLD)
        with pytest.raises(ValueError, match="another process group"):
            GraphedTrainStep(model, peer, batcher, 4, group=subs[1 - rank])
        # the engine's own group passes the group checks and stops at the CPU model
        with pytest.raises(ValueError, match="CUDA"):
            GraphedTrainStep(model, peer, batcher, 4, group=subs[rank])
        open(os.path.join(out, "ok%d" % rank), "w").write("ok")
    finally:
        dist.destroy_process_group()


def test_refusals_two_ranks(tmp_path):
    corpus = build_corpus(str(tmp_path / "corpus"), 8, 9000, 12000)
    mp.spawn(_worker, args=(2, _free_port(), corpus, str(tmp_path)), nprocs=2, join=True)
    assert all(os.path.exists(tmp_path / ("ok%d" % r)) for r in range(2))
