"""Product-side data-parallel test on 2 GPUs (skipped with fewer): the NCCL path of WaveNet.train_step — phased backward, one
all-reduce per layer group overlapped with the next group's weight-gradient GEMM — must give the same averaged gradients as ONE
GPU running the concatenated batch (wavenet.py:561-593: tower gradients are averaged, then clipped, then applied). Also Tacotron's
single all-reduce (tacotron.py:406-423). Needs two GPUs."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _wn_hp():
    from hparams import hparams
    hp = hparams.copy()
    hp.parse("input_type=mulaw-quantize,quantize_channels=256,out_channels=256,layers=6,stacks=2,residual_channels=128,"
             "gate_channels=256,skip_out_channels=128,upsample_scales=[4,4],hop_size=16,wavenet_dropout=0.0")
    return hp


def _wn_data(B, T):
    g = torch.Generator().manual_seed(7)
    idx = torch.randint(0, 256, (B, T), generator=g, dtype=torch.int32)
    c = torch.rand(B, 80, T // 16, generator=g)
    return idx, c, torch.full((B,), T, dtype=torch.int32)


def _worker(rank, world, port, out_path):
    import torch.distributed as dist
    from t2_import import t2
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    hp = _wn_hp()
    Bg, T = 2 * world, 512
    idx, c, lens = _wn_data(Bg, T)
    sl = slice(2 * rank, 2 * rank + 2)
    m = t2.wavenet.WaveNet(hp, 2, T, device=dev)
    m.init_variables(seed=11)
    args = (idx[sl].to(dev), c[sl].to(dev), idx[sl].to(dev), lens[sl].to(dev))
    m.capture(*args, overlap_groups=3)
    m.train_step(world_size=world)
    torch.cuda.synchronize()
    grads_overlap = (m.grads / world).cpu()
    # same thing through the un-phased path (one graph + one monolithic all-reduce)
    m2 = t2.wavenet.WaveNet(hp, 2, T, device=dev)
    m2.init_variables(seed=11)
    m2.capture(*args)
    m2.train_step(world_size=world)
    torch.cuda.synchronize()
    if rank == 0:
        torch.save({"overlap": grads_overlap, "mono": (m2.grads / world).cpu(), "loss": m.loss_value()}, out_path)
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_wavenet_dp2_overlapped_allreduce_matches_single_gpu(tmp_path):
    import torch.multiprocessing as mp
    from t2_import import t2
    out = str(tmp_path / "dp.pt")
    mp.spawn(_worker, args=(2, 29533, out), nprocs=2, join=True)
    r = torch.load(out)
    hp = _wn_hp()
    idx, c, lens = _wn_data(4, 512)
    single = t2.wavenet.WaveNet(hp, 4, 512)
    single.init_variables(seed=11)
    single.forward(idx.cuda(), c.cuda(), idx.cuda(), lens.cuda())
    single.backward()
    torch.cuda.synchronize()
    ref = single.grads.cpu()
    # phased + overlapped == monolithic, bit for bit up to fp32 atomics order in the bias sums
    rel_paths = (r["overlap"] - r["mono"]).norm() / r["mono"].norm()
    rel_single = (r["overlap"] - ref).norm() / ref.norm()
    print("DP2: overlapped vs monolithic all-reduce rel %.3g | DP2 vs one GPU on the concatenated batch rel %.3g" % (rel_paths, rel_single))
    assert rel_paths < 1e-5
    # the per-item arithmetic is identical; only the order of the fp32 position sums differs (one 4-item reduction vs 2 + 2 + NCCL)
    assert rel_single < 2e-3
    for name, off, shape in single.tensors:
        n = 1
        for d in shape:
            n *= d
        a, b = r["overlap"][off:off + n], ref[off:off + n]
        if b.norm() > 1e-7:
            assert (a - b).norm() / b.norm() < 2e-2, name
