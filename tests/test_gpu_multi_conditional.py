"""The latent pool's gradient under `DistributedDataParallel` with 2 ranks (base_trainer.py:102-104): each rank looks up its half
of the batch's indices -- one index on both ranks, one repeated -- and back-propagates through the generator; the pool
gradient that DDP's reducer averages must equal the single-process gradient of the whole batch, and rows no rank indexed stay
exactly zero.  Ranks as in tests/test_gpu_multi.py: one GPU each over NCCL, or both on cuda:0 over gloo."""
import importlib
import os
import sys

import pytest
import torch

from test_gpu_multi import _init

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INDICES = [5, 2, 5, 5]          # rank 0: [5, 2], rank 1: [5, 5]


def _pool_worker(rank, world, port_no, out_path):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP
    dev = _init(rank, world, port_no)
    pkg = importlib.import_module("3dhumangan_b200")
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    rng = importlib.import_module("3dhumangan_b200.rng")
    from oracle import port
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(gen_height=64, gen_width=64, render_height=8, render_width=8, num_steps=32, nerf_noise=0.5)
    B = len(INDICES)
    params = port.init_generator_params(cfg, seed=5, sigma_gain=200.0, sigma_bias=1.0)
    codes, _ = pkg.synthetic.make_appearance(B, cfg["dataset_length"], cfg["latent_dim"], seed=3)
    params["latent_pool.latents"] = codes
    cond = pkg.synthetic.make_conditions(B, seed=4)
    idx = torch.tensor(INDICES, dtype=torch.int64)
    torch.manual_seed(6)
    u, noise = rng.draw_render_noise(B, 64, cfg["num_steps"], "cpu", cfg["sample_dist"])
    wgt = torch.randn(B, 3, 64, 64, generator=torch.Generator().manual_seed(7))

    def run(sl, ddp):
        G = gen.Map3DGenerator(**cfg).to(dev)
        G.load_state_dict(params)
        G.set_device(dev)
        G.train()
        net = DDP(G, device_ids=[dev] if dist.get_backend() == "nccl" else None, find_unused_parameters=True,
                  broadcast_buffers=False) if ddp else G
        rng.draw_render_noise = lambda *a, **k: (u[sl].to(dev), noise[sl].to(dev))
        z = torch.zeros(sl.stop - sl.start, cfg["latent_dim"], device=dev)        # replaced by the pool rows
        out = net(z, {k: v[sl].to(dev) for k, v in cond.items()}, latent_indices=idx[sl].to(dev), **cfg)
        ((out["rgbs"] * wgt[sl].to(dev)).sum() / out["rgbs"].shape[0]).backward()      # DDP averages the per-rank losses
        return G.latent_pool.latents.grad.cpu()

    half = B // world
    dp = run(slice(rank * half, (rank + 1) * half), True)
    torch.cuda.synchronize()
    both = [None, None]
    dist.all_gather_object(both, dp)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        single = run(slice(0, B), False)
        torch.save({"dp": both, "single": single}, out_path)


def test_ddp_pool_gradient_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    out = str(tmp_path / "pool.pt")
    mp.spawn(_pool_worker, args=(2, 29800 + os.getpid() % 90, out), nprocs=2, join=True)
    r = torch.load(out)
    dp0, dp1 = r["dp"]
    single = r["single"]
    assert torch.equal(dp0, dp1)                                  # all-reduced: identical on both ranks
    touched = torch.zeros(single.shape[0], dtype=torch.bool)
    touched[INDICES] = True
    assert not dp0[~touched].any() and not single[~touched].any()
    for row in sorted(set(INDICES)):
        ref = single[row].double()
        err = float((dp0[row].double() - ref).norm() / ref.norm())
        # same arithmetic up to the SyncBatchNorm reduction order and LeakyReLU-mask flips (tests/test_gpu_multi.py); a
        # gradient that DDP did not see, or one rank's contribution to row 5 missing, is off by O(1)
        assert err < 2e-2, (row, err)
