"""GPU tests that need TWO devices (skipped on a machine with one GPU; run with `python -m pytest tests/test_multi_gpu.py -m gpu`
on two).

* a model living on cuda:1 while cuda:0 is the current device (ADVICE r1: nothing selected the device) gives the
  same result as on cuda:0 -- the reference's `.to(device)` works on any device;
* `shard.run_sharded` (BASELINE config[2] host logic) over NCCL, world size 2, one process per GPU: every sequence's
  predictions equal the single-process result."""
import os
import socket

import pytest
import torch

from conftest import get_state_dict, rel_l2

pytestmark = pytest.mark.gpu


def _two_gpus():
    return torch.cuda.is_available() and torch.cuda.device_count() >= 2


@pytest.mark.skipif(not _two_gpus(), reason="needs 2 GPUs")
def test_model_on_second_device_while_first_is_current():
    from spann3r_b200 import Spann3R, synth
    torch.cuda.set_device(0)
    frames = synth.make_frames(3, 224, 224)
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        m = Spann3R(dus3r_name=None)
        m.load_state_dict(get_state_dict(True), strict=True)
        m = m.to(dev).eval()
        assert torch.cuda.current_device() == 0
        preds, _ = m(frames)
        torch.cuda.synchronize(dev)
        assert all(v.device == torch.device(dev) for p in preds for v in p.values())
        outs.append([{k: v.cpu() for k, v in p.items()} for p in preds])
        del m
    for a, b in zip(*outs):
        for k in a:
            assert torch.equal(a[k], b[k]), k          # same kernels, same tile plans: bit-identical across devices


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from spann3r_b200 import Spann3R, shard, synth
    from conftest import get_state_dict as gsd
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(gsd(True), strict=True)
    m = m.to(f"cuda:{rank}").eval()
    seqs = [synth.make_frames(3, 224, 224, seed0=100 * s + 1) for s in range(5)]
    out = shard.run_sharded(lambda fr: m(fr), seqs, per_gpu_batch=2)
    ms = shard.max_over_ranks(10.0 + rank, device=torch.device("cuda", rank))
    ret[rank] = ({i: [{k: v.cpu() for k, v in p.items()} for p in preds] for i, preds in out.items()}, ms)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(not _two_gpus(), reason="needs 2 GPUs")
def test_run_sharded_nccl_two_ranks_equals_single_process():
    import torch.multiprocessing as mp
    from spann3r_b200 import Spann3R, synth
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    got = {}
    for r in range(world):
        part, ms = ret[r]
        assert ms == 11.0                                     # max over ranks of (10 + rank)
        assert sorted(part) == list(range(r, 5, world))       # round-robin deal
        got.update(part)
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(get_state_dict(True), strict=True)
    m = m.cuda().eval()
    for s in range(5):
        preds, _ = m(synth.make_frames(3, 224, 224, seed0=100 * s + 1))
        for p, q in zip(preds, got[s]):
            for k in p:
                assert rel_l2(q[k], p[k].cpu()) < 1e-4, (s, k)   # B = 2 lockstep vs B = 1: other tile shapes


def _ddp_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from spann3r_b200 import Spann3R, synth
    from conftest import get_state_dict as gsd
    m = Spann3R(dus3r_name=None, memory_dropout=0.0)
    m.load_state_dict(gsd(True), strict=True)
    m = m.to(f"cuda:{rank}").train()
    ddp = torch.nn.parallel.DistributedDataParallel(m, device_ids=[rank], find_unused_parameters=True, static_graph=True)
    frames = synth.make_frames(3, 224, 224, seed0=1 + 100 * rank)     # a different sequence per rank
    preds, _ = ddp(frames)
    loss = sum((p["conf"].log().mean() + p[k].square().mean()) for p in preds for k in p if k != "conf")
    loss.backward()
    named = dict(m.named_parameters())
    keys = ["dust3r.enc_blocks.0.attn.qkv.weight", "dust3r.dec_blocks.11.mlp.fc2.weight", "value_out.weight", "norm_q.weight"]
    ret[rank] = {k: named[k].grad.detach().cpu() for k in keys}
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(not _two_gpus(), reason="needs 2 GPUs")
def test_ddp_allreduces_the_recompute_backward_gradients():
    """SURVEY.md §8e-train: `DistributedDataParallel` around the training-mode model (the reference's wrap,
    spann3r/training.py:322-325) averages the gradients of the two ranks over NCCL: identical on both ranks afterwards and
    equal to the mean of the single-process gradients of the two sequences."""
    import torch.multiprocessing as mp
    from spann3r_b200 import Spann3R, synth
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_ddp_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    for k in ret[0]:
        assert torch.equal(ret[0][k], ret[1][k]), k
    m = Spann3R(dus3r_name=None, memory_dropout=0.0)
    m.load_state_dict(get_state_dict(True), strict=True)
    m = m.cuda().train()
    named = dict(m.named_parameters())
    acc = {k: 0 for k in ret[0]}
    for r in range(world):
        m.zero_grad(set_to_none=True)
        preds, _ = m(synth.make_frames(3, 224, 224, seed0=1 + 100 * r))
        sum((p["conf"].log().mean() + p[k].square().mean()) for p in preds for k in p if k != "conf").backward()
        for k in acc:
            acc[k] = acc[k] + named[k].grad.detach().cpu() / world
    for k in acc:
        assert rel_l2(ret[0][k], acc[k]) < 2e-4, k      # cuDNN / cuBLAS backward kernels are not run-to-run deterministic (measured 3e-5)
