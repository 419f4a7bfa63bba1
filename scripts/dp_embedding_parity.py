"""N-GPU data-parallel parity of the token-embedding training steps (run under torchrun). Each rank
trains on its own sample, with its own prompt ids; after 4 steps the LoRA factors, the claimed
embedding rows and their AdamW moments (arena p / m / v), the slot list and the embedding table must
equal those of ONE process that runs the concatenated batch (bs = world), and every rank must hold a
bitwise identical replica. Covers LoraEmbeddingStep in mode "table" and mode "placeholders" (with
unfreeze_lora_step crossed inside the run), eager and captured, and TextualInversionStep (eager).
The exchange is the NVLink peer path unless LB_DP_NCCL=1 (NCCL all-reduce + all-gathered ids).
Tiny host models, dropout 0, external noise.

    torchrun --nproc-per-node 2 scripts/dp_embedding_parity.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

import lora_b200 as L
from lora_b200.host.clip import build_text_encoder
from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
from lora_b200.train import LoraEmbeddingStep, StepConfig, TextualInversionStep

STEPS, HW, S = 4, 16, 77
TOL = 5e-3


def models(dev, lora=True):
    torch.manual_seed(0)
    unet = UNet2DConditionModel(UNetConfig.tiny()).to(dev)
    text = build_text_encoder(tiny=True).to(dev)
    unet.requires_grad_(False); text.requires_grad_(False)
    if lora:
        L.inject_trainable_lora(unet, r=4)
        L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
        g = torch.Generator(device=dev).manual_seed(1)
        for m in list(unet.modules()) + list(text.modules()):
            if type(m).__name__ == "LoraInjectedLinear":
                m.lora_up.weight.data.normal_(0, 0.05, generator=g)
    return unet, text


def sample(r, step, V, ph, world, dev):
    """Rank r's sample of `step`: overlapping per-rank id pools (tokens seen on one rank only, tokens
    shared), placeholder 0 on rank 0, placeholder 1 on the last rank."""
    g = torch.Generator().manual_seed(1000 + 10 * step + r)
    ids = torch.randint(20 * r, 20 * r + 60, (1, S), generator=g)
    if r == 0:
        ids[0, 2] = ph[0]
    if r == world - 1:
        ids[0, 4] = ph[1]
    return (torch.randn(1, 4, HW, HW, generator=g) * 0.18215, ids, torch.randn(1, 4, HW, HW, generator=g),
            torch.randint(0, 800, (1,), generator=g))


def cfg_of(mode, graph, peer=True):
    common = dict(use_cuda_graph=graph, autocast_dtype=torch.bfloat16, external_noise=True, peer_allreduce=peer,
                  lr_scheduler="linear", max_train_steps=8)
    if mode == "table":
        return StepConfig(t_multiplier=0.8, lr_step_first=True, adam_weight_decay=1e-3, **common)
    if mode == "placeholders":
        return StepConfig(adam_weight_decay=1e-2, learning_rate_text=5e-5, **common)
    return StepConfig(lr_scheduler="constant", **{k: v for k, v in common.items() if k != "lr_scheduler"})


def make(kind, bs, dev, graph=False, peer=True):
    lora = kind != "ti"
    unet, text = models(dev, lora)
    V = text.get_input_embeddings().weight.shape[0]
    ph = [V - 2, V - 1]
    shape = (bs, 4, HW, HW)
    if kind == "ti":
        return TextualInversionStep(unet, text, ph, cfg_of(kind, False, peer), lr=5e-3, latent_shape=shape,
                                    device=dev), text, ph
    kw = dict(unfreeze_lora_step=2) if kind == "placeholders" else {}
    return LoraEmbeddingStep(unet, text, ph, cfg_of(kind, graph, peer), lr_embedding=1e-3, mode=kind,
                             row_capacity=256, latent_shape=shape, device=dev, **kw), text, ph


def run(st, text, ph, ranks, world, dev):
    V = text.get_input_embeddings().weight.shape[0]
    for step in range(STEPS):
        parts = [sample(r, step, V, ph, world, dev) for r in ranks]
        lat, ids, noise, t = (torch.cat([p[i] for p in parts]).to(dev) for i in range(4))
        st.latents.copy_(lat); st.input_ids.copy_(ids); st.noise.copy_(noise); st.timesteps.copy_(t)
        st.step_device()
    torch.cuda.synchronize()
    if hasattr(st, "rows"):
        st.flush()
        a = st.arena
        out = {"p": a.p, "m": a.m, "v": a.v, "slot_tok": st.rows.slot_tokens()}
    else:
        out = {"p": st.ti.rows.data, "m": st.ti.m, "v": st.ti.v}
    out["table"] = text.get_input_embeddings().weight.detach()
    return {k: v.detach().clone() for k, v in out.items()}


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ["NCCL_DEBUG"] = "WARN"
    peer = os.environ.get("LB_DP_NCCL", "0") != "1"
    kinds = [("table", False), ("table", True), ("placeholders", False), ("placeholders", True), ("ti", False)]
    # (b) first, before the process group exists: one process running the concatenated batch (bs = world)
    single = {}
    for kind in ("table", "placeholders", "ti"):
        st, text, ph = make(kind, world, dev)
        single[kind] = run(st, text, ph, list(range(world)), world, dev)
        if hasattr(st, "release"):
            st.release()
        del st
    dist.init_process_group("nccl", device_id=dev)
    worst, exchange = 0.0, None
    for kind, graph in kinds:
        st, text, ph = make(kind, 1, dev, graph=graph, peer=peer)
        if graph:
            st.prepare()
            assert st.graph is not None, st.graph_error
        if kind != "ti" and world == 1:
            exchange = "none (one rank)"
        elif kind != "ti":
            exchange = "nvlink-peer (lb_optim_step_dp + lb_embed_rows_scatter_dp)" if st.peer_allreduce else \
                "nccl (all-reduce + all-gathered ids)"
        got = run(st, text, ph, [rank], world, dev)
        want = single[kind]
        errs = {k: rel(got[k], want[k]) for k in ("p", "m", "v", "table")}
        slots_ok = kind == "ti" or torch.equal(got["slot_tok"], want["slot_tok"])
        same = True                              # bitwise identical replicas
        for k, v in got.items():
            if k == "slot_tok":
                n = torch.tensor([v.numel()], device=dev)
                dist.broadcast(n, src=0)
                if int(n) != v.numel():
                    same = False
                    continue
            ref = v.clone()
            dist.broadcast(ref, src=0)
            same = same and torch.equal(ref, v)
        flags = torch.tensor([max(errs.values()), 0.0 if slots_ok else 1.0, 0.0 if same else 1.0], device=dev)
        dist.all_reduce(flags, op=dist.ReduceOp.MAX)
        worst = max(worst, float(flags[0]))
        if rank == 0:
            print(f"dp_embedding_parity world={world} step={kind} {'captured' if graph else 'eager'} "
                  f"rel_err p/m/v/table=" + "/".join(f"{errs[k]:.2e}" for k in ("p", "m", "v", "table")) +
                  f" slot_tok_equal={float(flags[1]) == 0.0} replicas_identical={float(flags[2]) == 0.0}", flush=True)
        assert float(flags[0]) < TOL and float(flags[1]) == 0.0 and float(flags[2]) == 0.0, (kind, graph)
        if hasattr(st, "release"):
            st.release()
        del st
    if rank == 0:
        print(f"dp_embedding_parity world={world} exchange={exchange} worst_rel_err={worst:.2e}")
        print("dp_embedding_parity OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
