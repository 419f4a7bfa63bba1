"""N > 1 host logic on CPU with the gloo backend, world_size 2 (the data path has exactly one
collective: a SUM all-reduce of the flat LoRA gradient buffer, lora_b200/dist.py)."""
import os
import socket

import torch
import torch.multiprocessing as mp

from lora_b200.dist import shard_indices


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from lora_b200.dist import allreduce_sum_, world_info
    from oracle import lora_ops as O
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    assert world_info() == (rank, world)
    torch.manual_seed(0)
    p0 = torch.randn(1000)                     # identical replica on every rank (same seed)
    torch.manual_seed(100 + rank)
    g_local = torch.randn(1000) * 3            # per-rank gradient from its own shard
    flat = g_local.clone()
    ws = allreduce_sum_(flat)
    assert ws == world
    # fused step semantics: g_sum with inv_world = 1/world  (clip on the AVERAGED gradient)
    new_p, _, _, total = O.clip_adamw_step([p0], [flat], [torch.zeros(1000)], [torch.zeros(1000)],
                                           1, [1e-3], inv_world=1.0 / world)
    torch.save({"p": new_p[0], "g_local": g_local, "total": total}, os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_allreduce_then_step_equals_single_process_on_mean_gradient(tmp_path):
    world = 2
    port = _free_port()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    from oracle import lora_ops as O
    outs = [torch.load(tmp_path / f"r{r}.pt") for r in range(world)]
    assert torch.equal(outs[0]["p"], outs[1]["p"])            # replicas stay in lock-step
    g_mean = (outs[0]["g_local"] + outs[1]["g_local"]) / world
    torch.manual_seed(0)
    p0 = torch.randn(1000)
    want, _, _, total = O.clip_adamw_step([p0], [g_mean], [torch.zeros(1000)], [torch.zeros(1000)], 1, [1e-3])
    assert torch.allclose(outs[0]["p"], want[0], rtol=0, atol=1e-12)
    assert abs(outs[0]["total"] - total) < 1e-9


def test_shard_indices_round_robin():
    assert shard_indices(9, 0, 2) == [0, 2, 4, 6, 8]
    assert shard_indices(9, 1, 2) == [1, 3, 5, 7, 1]           # padded by wrapping: equal step counts
    assert shard_indices(9, 1, 2, drop_last=True) == [1, 3, 5, 7]
    assert shard_indices(4, 3, 8) == [3]
    for world in (1, 2, 4, 8):
        lens = {len(shard_indices(10, r, world)) for r in range(world)}
        assert len(lens) == 1
        seen = set()
        for r in range(world):
            seen.update(shard_indices(10, r, world))
        assert seen == set(range(10))


def _cpu_svd_stub(W_tuned, W_base, rank, power_iters=1, clamp_quantile=None, seed=0):
    """Exact truncated SVD (+ the reference's quantile clamp) on CPU standing in for the CUDA call
    (same return contract as lora_b200.svd.svd_lowrank_ragged): the test below is about WHICH
    process distils WHICH site and how the factors travel, not about the factorisation."""
    ups, downs, sig, his = [], [], [], []
    for wt, wb in zip(W_tuned, W_base):
        U, S, Vh = torch.linalg.svd(wt.float() - wb.float(), full_matrices=False)
        u, d = U[:, :rank] * S[:rank], Vh[:rank]
        if clamp_quantile is not None:
            hi = torch.quantile(torch.cat([u.flatten(), d.flatten()]), clamp_quantile)
            u, d = u.clamp(-hi, hi), d.clamp(-hi, hi)
            his.append(hi)
        ups.append(u)
        downs.append(d)
        sig.append(S[:rank])
    return ups, downs, sig, his


def _build_pair():
    import copy
    import lora_b200 as L
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    torch.manual_seed(0)
    base = UNet2DConditionModel(UNetConfig.tiny())
    tuned = copy.deepcopy(base)
    g = torch.Generator().manual_seed(1)
    for prm in tuned.parameters():
        if prm.dim() >= 2:
            prm.data.add_(torch.randn(prm.shape, generator=g) * 0.01)
    L.inject_trainable_lora_extended(base, r=4)
    L.inject_trainable_lora_extended(tuned, r=4)
    return base, tuned


def _factors(model):
    return [t.detach().clone() for m in model.modules() if type(m).__name__.startswith("LoraInjected")
            for t in (m.lora_up.weight, m.lora_down.weight)]


def _svd_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    import lora_b200.svd as svd
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    seen = []
    def stub(W_tuned, W_base, r, power_iters=1, clamp_quantile=None, seed=0):
        seen.append(len(W_tuned))
        return _cpu_svd_stub(W_tuned, W_base, r, power_iters, clamp_quantile)
    svd.svd_lowrank_ragged = stub
    base, tuned = _build_pair()
    svd.overwrite_base(base, tuned, rank=4, clamp_quantile=0.99, shard=(rank, world))
    torch.save({"factors": _factors(base), "n_done": sum(seen)}, os.path.join(out_dir, f"svd{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_svd_distill_equals_single_process(tmp_path):
    """SVD distillation on several GPUs: weight deltas are sharded round-robin over the
    ranks (no collective on the compute path), factors exchanged by one all-reduce over a
    zero-padded flat buffer; every rank must end with exactly the single-process result."""
    import lora_b200.svd as svd
    world = 2
    mp.spawn(_svd_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [torch.load(tmp_path / f"svd{r}.pt") for r in range(world)]
    real = svd.svd_lowrank_ragged
    try:
        svd.svd_lowrank_ragged = _cpu_svd_stub
        base, tuned = _build_pair()
        svd.overwrite_base(base, tuned, rank=4, clamp_quantile=0.99)
    finally:
        svd.svd_lowrank_ragged = real
    want = _factors(base)
    n_sites = len(want) // 2
    assert outs[0]["n_done"] + outs[1]["n_done"] == n_sites and abs(outs[0]["n_done"] - outs[1]["n_done"]) <= 1
    for r in range(world):
        got = outs[r]["factors"]
        assert len(got) == len(want)
        assert all(torch.equal(a, b) for a, b in zip(got, want)), r
