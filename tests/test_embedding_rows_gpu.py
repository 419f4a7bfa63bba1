"""On the GPU: the token-embedding table trained together with the LoRA factors
(lora_b200/embed_rows.py, lora_b200.train.LoraEmbeddingStep) -- the gradient scatter against a dense
index_add_, the lazy decay against torch.optim.AdamW over the whole table, the slot overflow, both
reference configurations against oracle/joint_ref.py, and the captured step."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _text_arena(cap=64, lr_rows=1e-3, placeholders=(998,), weight_decay=1e-2, mode="table"):
    """A tiny text encoder with LoRA sites, an arena with a rows group, and its EmbeddingRows."""
    import lora_b200 as L
    from lora_b200.arena import LoraArena
    from lora_b200.embed_rows import EmbeddingRows
    from lora_b200.host.clip import build_text_encoder
    torch.manual_seed(0)
    te = build_text_encoder(tiny=True).to(DEV)
    te.requires_grad_(False)
    L.inject_trainable_lora(te, target_replace_module={"CLIPAttention"}, r=4)
    D = te.get_input_embeddings().weight.shape[1]
    arena = LoraArena([(te, 1e-4)], device=torch.device(DEV), rows=(cap, D, lr_rows))
    rows = EmbeddingRows(te, arena, list(placeholders), mode=mode, weight_decay=weight_decay)
    return te, arena, rows


def test_arena_rows_group_is_appended_after_the_lora_groups():
    import lora_b200 as L
    from lora_b200.arena import LoraArena
    from lora_b200.host.clip import build_text_encoder
    te = build_text_encoder(tiny=True).to(DEV)
    te.requires_grad_(False)
    L.inject_trainable_lora(te, target_replace_module={"CLIPAttention"}, r=4)
    plain = LoraArena([(te, 1e-4)], device=torch.device(DEV))
    wide = LoraArena([(te, 1e-4)], device=torch.device(DEV), rows=(100, 48, 5e-3))
    assert plain.rows_group is None and len(plain.base_lr) == 1
    assert wide.group_off[:2] == plain.group_off and wide.rows_group == 1
    assert wide.n == plain.n + 100 * 48 and wide.base_lr == [1e-4, 5e-3]
    assert torch.equal(wide.table, plain.table)
    assert wide.rows_view(wide.p).shape == (100, 48)


@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
def test_scatter_matches_dense_index_add_and_is_deterministic(gdtype):
    te, arena, rows = _text_arena()
    V, D = rows.V, rows.D
    g = torch.Generator(device=DEV).manual_seed(1)
    ids = torch.randint(0, 40, (2, 77), device=DEV, generator=g)       # many repeats
    ids[0, 3], ids[1, 50] = 998, 998                                     # the placeholder
    grad = torch.randn(2, 77, D, device=DEV, generator=g).to(gdtype)
    snap = rows.snapshot()
    rows._scatter(ids, grad)
    torch.cuda.synchronize()
    dense = torch.zeros(V, D, dtype=torch.float64, device=DEV)
    dense.index_add_(0, ids.reshape(-1), grad.reshape(-1, D).double())
    toks = rows.slot_tok[: int(rows.state[1])].long()
    got = arena.rows_view(arena.g)[: toks.numel()].double()
    want = dense[toks]
    assert float((got - want).norm() / want.norm()) < 1e-6
    assert set(toks.tolist()) == set(ids.reshape(-1).tolist())
    # slots: the placeholder first (claimed at construction), then first-occurrence order
    order = [998] + [t for i, t in enumerate(ids.reshape(-1).tolist()) if t not in ids.reshape(-1).tolist()[:i] and t != 998]
    assert toks.tolist() == order
    first_g = arena.rows_view(arena.g).clone()
    first_slots = rows.slot_of.clone()
    # a second identical launch from the same state is bitwise identical
    arena.g.zero_()
    rows.restore(snap)
    rows._scatter(ids, grad)
    torch.cuda.synchronize()
    assert torch.equal(arena.rows_view(arena.g), first_g) and torch.equal(rows.slot_of, first_slots)
    # a second batch after the write-back commits the claims: new tokens follow, in order
    rows.write_back()
    ids2 = torch.tensor([[45, 998, 41, 45, 40] + [998] * 72], device=DEV)
    rows._scatter(ids2, torch.randn(1, 77, D, device=DEV).to(gdtype))
    torch.cuda.synchronize()
    assert rows.slot_tok[: int(rows.state[1])].tolist() == order + [45, 41, 40]
    assert int(rows.state[3]) == 0


def test_lazy_decay_equals_dense_adamw_on_the_whole_table():
    wd, lr0, steps = 1e-2, 1e-2, 6
    te, arena, rows = _text_arena(cap=128, lr_rows=lr0, placeholders=(999,), weight_decay=wd)
    table = te.get_input_embeddings().weight
    V, D = table.shape
    table0 = table.detach().clone()
    dense = torch.nn.Parameter(table.detach().clone().float())
    opt = torch.optim.AdamW([dense], lr=lr0, weight_decay=wd)
    g = torch.Generator(device=DEV).manual_seed(2)
    late = 700                                           # first seen at step 4
    seen = {999}
    for k in range(steps):
        lr_k = lr0 * (steps - k) / steps                 # linear schedule
        pool = torch.arange(10 * k, 10 * k + 30, device=DEV)
        ids = pool[torch.randint(0, 30, (1, 77), device=DEV, generator=g)]
        if k == 4:
            ids[0, 7] = late
        seen |= set(ids.reshape(-1).tolist())
        grad = torch.randn(1, 77, D, device=DEV, generator=g) * 0.1
        rows._scatter(ids, grad)
        arena.set_lr([1e-4, lr_k])
        arena.step(weight_decay=wd, max_norm=1.0)
        rows.write_back()
        dg = torch.zeros(V, D, device=DEV)
        dg.index_add_(0, ids.reshape(-1), grad.reshape(-1, D))
        dense.grad = dg
        torch.nn.utils.clip_grad_norm_([dense], 1.0)
        opt.param_groups[0]["lr"] = lr_k
        opt.step()
    assert late in rows.slot_tokens().tolist()
    rows.flush()
    torch.cuda.synchronize()
    got, want = table.detach().double(), dense.detach().double()
    assert float((got - want).norm() / want.norm()) < 1e-6
    never = torch.ones(V, dtype=torch.bool, device=DEV)
    never[list(seen)] = False
    assert float((got[never] - want[never]).norm() / want[never].norm()) < 1e-6
    assert not torch.equal(got[never], table0[never].double())           # they did decay
    assert float(rows.decay) == 1.0


def test_overflow_is_flagged_and_leaves_claimed_rows_alone():
    from lora_b200._C import LoraB200Error
    te, arena, rows = _text_arena(cap=8, placeholders=(999,))
    D = rows.D
    first = torch.tensor([[5, 6, 7] * 25 + [5, 6]], device=DEV)
    rows._scatter(first, torch.randn(1, 77, D, device=DEV))
    arena.step(weight_decay=1e-2)
    rows.write_back()
    rows.check()
    before_master = arena.rows_view(arena.p)[:4].clone()
    before_slots = rows.slot_of[[999, 5, 6, 7]].clone()
    ids = torch.arange(100, 120, device=DEV).repeat(4)[:77].reshape(1, 77)   # 20 new distinct tokens
    rows._scatter(ids, torch.randn(1, 77, D, device=DEV))
    torch.cuda.synchronize()
    with pytest.raises(LoraB200Error):
        rows.check()
    with pytest.raises(LoraB200Error):
        rows.flush()
    assert int(rows.state[1]) == 8                                      # filled to capacity, no further
    assert torch.equal(rows.slot_of[[999, 5, 6, 7]], before_slots)
    assert torch.equal(arena.rows_view(arena.p)[:4], before_master)
    assert rows.slot_of[100:104].tolist() == [4, 5, 6, 7] and int((rows.slot_of[104:120] >= 0).sum()) == 0


def _joint_models(seed=0):
    import lora_b200 as L
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from oracle.ref_modules import ref_inject
    torch.manual_seed(seed)
    unet = UNet2DConditionModel(UNetConfig.tiny()).to(DEV)
    text = build_text_encoder(tiny=True).to(DEV)
    unet.requires_grad_(False)
    text.requires_grad_(False)
    unet_r, text_r = copy.deepcopy(unet), copy.deepcopy(text)
    L.inject_trainable_lora(unet, r=4)
    L.inject_trainable_lora(text, target_replace_module={"CLIPAttention"}, r=4)
    us = ref_inject(unet_r, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text_r, {"CLIPAttention"}, r=4)
    ours = [m for m in list(unet.modules()) + list(text.modules()) if type(m).__name__ == "LoraInjectedLinear"]
    g = torch.Generator(device=DEV).manual_seed(3)
    for o, r in zip(ours, us + ts):
        o.lora_up.weight.data.normal_(0, 0.05, generator=g)
        r.up.data.copy_(o.lora_up.weight.data)
        r.down.data.copy_(o.lora_down.weight.data)
    return unet, text, unet_r, text_r, us, ts


def _batches(n, V, tok, seed=8):
    gi = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for _ in range(n):
        lat = torch.randn(2, 4, 16, 16, device=DEV, generator=gi) * 0.18215
        ids = torch.randint(0, 60, (2, 77), device=DEV, generator=gi)     # a small pool: rows repeat across steps
        ids[0, 2], ids[1, 5] = tok[0], tok[1]
        noise = torch.randn(2, 4, 16, 16, device=DEV, generator=gi)
        t = torch.randint(0, 800, (2,), device=DEV, generator=gi)
        out.append((lat, ids, noise, t))
    return out


def _factors(step):
    return step.arena.p[: step.arena.group_off[step.arena.rows_group]].clone()


def test_mode_table_matches_oracle_continue_inversion():
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraEmbeddingStep, StepConfig
    from oracle.joint_ref import RefJointStep
    unet, text, unet_r, text_r, us, ts = _joint_models()
    V = text.get_input_embeddings().weight.shape[0]
    tok = [V - 2, V - 1]
    lr, lr_text, lr_emb, wd = 1e-4, 1e-5, 5e-5, 1e-3
    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16, t_multiplier=0.8, lr_step_first=True,
                     lr_scheduler="linear", max_train_steps=6, learning_rate=lr, learning_rate_text=lr_text,
                     adam_weight_decay=wd, external_noise=True)
    eng = LoraEmbeddingStep(unet, text, tok, cfg, lr_embedding=lr_emb, mode="table", latent_shape=(2, 4, 16, 16))
    ref = RefJointStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, "table", lr=lr, lr_text=lr_text,
                       lr_embedding=lr_emb, lr_lambda=lambda k: max(0.0, 1.0 - k / 6), weight_decay=wd,
                       t_multiplier=0.8, autocast_dtype=torch.bfloat16)
    table0 = text.get_input_embeddings().weight.detach().clone()
    seen = set(tok)
    for lat, ids, noise, t in _batches(3, V, tok):
        seen |= set(ids.reshape(-1).tolist())
        l_ref = float(ref.step(lat, ids, noise, t))
        eng.latents.copy_(lat); eng.input_ids.copy_(ids); eng.noise.copy_(noise); eng.timesteps.copy_(t)
        l_ours = float(eng.step_device())
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (l_ours, l_ref)
        got = text.get_input_embeddings().weight.detach().double()
        want = ref.table.detach().double()
        s = torch.tensor(sorted(seen), device=DEV)
        assert float((got[s] - want[s]).norm() / want[s].norm()) < 1e-3
        d_ours, d_ref = got[s] - table0[s].double(), want[s] - table0[s].double()
        assert float((d_ours * d_ref).sum() / (d_ours.norm() * d_ref.norm())) > 0.95   # the same update
    eng.flush()
    got = text.get_input_embeddings().weight.detach().double()
    want = ref.table.detach().double()
    unseen = torch.ones(V, dtype=torch.bool, device=DEV)
    unseen[sorted(seen)] = False
    assert float((got[unseen] - want[unseen]).norm() / want[unseen].norm()) < 1e-6
    assert not torch.equal(got[unseen], table0[unseen].double())          # they did decay
    eng.release()


def test_mode_placeholders_matches_oracle_train_lora_w_ti():
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.train import LoraEmbeddingStep, StepConfig
    from oracle.joint_ref import RefJointStep
    unet, text, unet_r, text_r, us, ts = _joint_models(seed=1)
    emb = text.get_input_embeddings()
    V = emb.weight.shape[0]
    tok = [V - 2, V - 1]
    lr, lr_text, lr_ti, wd = 1e-4, 5e-5, 5e-4, 1e-2
    cfg = StepConfig(use_cuda_graph=False, autocast_dtype=torch.bfloat16, lr_scheduler="linear",
                     max_train_steps=8, learning_rate=lr, learning_rate_text=lr_text, adam_weight_decay=wd,
                     external_noise=True)
    eng = LoraEmbeddingStep(unet, text, tok, cfg, lr_embedding=lr_ti, mode="placeholders", unfreeze_lora_step=2,
                            latent_shape=(2, 4, 16, 16))
    ref = RefJointStep(unet_r, text_r, DDPMNoiser(device=DEV), us, ts, "placeholders", lr=lr, lr_text=lr_text,
                       lr_embedding=lr_ti, lr_lambda=lambda k: max(0.0, 1.0 - k / 8), weight_decay=wd,
                       autocast_dtype=torch.bfloat16, placeholder_token_ids=tok, unfreeze_lora_step=2)
    table0 = emb.weight.detach().clone()
    others = torch.ones(V, dtype=torch.bool, device=DEV)
    others[tok] = False
    for k, (lat, ids, noise, t) in enumerate(_batches(4, V, tok, seed=9)):
        f0, rows0 = _factors(eng), emb.weight.detach()[tok].clone()
        l_ref = float(ref.step(lat, ids, noise, t))
        eng.latents.copy_(lat); eng.input_ids.copy_(ids); eng.noise.copy_(noise); eng.timesteps.copy_(t)
        l_ours = float(eng.step_device())
        torch.cuda.synchronize()
        assert abs(l_ours - l_ref) < 1e-2 * abs(l_ref), (k, l_ours, l_ref)
        f1, rows1 = _factors(eng), emb.weight.detach()[tok]
        if k < 2:
            assert torch.equal(f1, f0) and not torch.equal(rows1, rows0), k
        else:
            assert torch.equal(rows1, rows0) and not torch.equal(f1, f0), k
        assert torch.equal(emb.weight.detach()[others], table0[others])
        # Adam's first updates are close to lr * sign(g): an element whose gradient is near zero can flip
        # sign under bf16 autocast and cost 2 * lr, so compare the rows loosely and their updates by direction
        want = ref.table.detach()[tok].double()
        assert float((rows1.double() - want).norm() / want.norm()) < 2e-2, k
        d_ours, d_ref = rows1.double() - table0[tok].double(), want - table0[tok].double()
        assert float((d_ours * d_ref).sum() / (d_ours.norm() * d_ref.norm())) > 0.95, k
    eng.release()
    assert torch.equal(emb.weight.detach()[others], table0[others])


def test_captured_joint_step_matches_eager_and_prepare_restores_state():
    from lora_b200 import ops
    from lora_b200.train import LoraEmbeddingStep, LoraTrainStep, StepConfig

    def make(graph, seed=0, joint=True):
        unet, text, *_ = _joint_models(seed)
        V = text.get_input_embeddings().weight.shape[0]
        cfg = StepConfig(use_cuda_graph=graph, autocast_dtype=torch.bfloat16, t_multiplier=0.8, lr_step_first=True,
                         lr_scheduler="linear", max_train_steps=10, adam_weight_decay=1e-3, external_noise=True)
        if not joint:
            return LoraTrainStep(unet, text, cfg, latent_shape=(2, 4, 16, 16)), text
        return LoraEmbeddingStep(unet, text, [V - 2, V - 1], cfg, lr_embedding=1e-3, mode="table",
                                 latent_shape=(2, 4, 16, 16)), text

    plain, _ = make(False, joint=False)
    eager, te_e = make(False)
    graph, te_g = make(True)
    V = te_e.get_input_embeddings().weight.shape[0]
    batches = _batches(4, V, [V - 2, V - 1], seed=11)
    # launches per step: the plain step's plus the scatter and the write-back
    counts = []
    for st in (plain, eager):
        lat, ids, noise, t = batches[0]
        st.latents.copy_(lat); st.input_ids.copy_(ids); st.noise.copy_(noise); st.timesteps.copy_(t)
        st._body()
        ops.LAUNCH_COUNT = 0
        st._body()
        counts.append(ops.LAUNCH_COUNT)
    assert counts[1] == counts[0] + 2, counts
    del plain
    # prepare() on the graph engine leaves every piece of state where it found it
    graph.latents.copy_(batches[0][0]); graph.input_ids.copy_(batches[0][1])
    graph.noise.copy_(batches[0][2]); graph.timesteps.copy_(batches[0][3])
    before = graph._snapshot()
    graph.prepare()
    assert graph.graph is not None and graph.graph_error is None
    after = graph._snapshot()
    for key in ("p", "m", "v", "step"):
        assert torch.equal(before[key], after[key]), key
    for key in ("table", "slot_of", "slot_tok", "state", "decay"):
        assert torch.equal(before["rows"][key], after["rows"][key]), key
    # the eager engine ran two bodies above: bring it back to the construction state of the graph engine
    init = _snapshot_like(graph, before)
    eager._restore(init)
    for lat, ids, noise, t in batches:
        outs = []
        for st in (eager, graph):
            st.latents.copy_(lat); st.input_ids.copy_(ids); st.noise.copy_(noise); st.timesteps.copy_(t)
            outs.append(float(st.step_device()))
        torch.cuda.synchronize()
        assert abs(outs[0] - outs[1]) < 2e-3 * abs(outs[0]), outs
    assert float((_factors(eager) - _factors(graph)).abs().max()) < 1e-4
    ge, gg = te_e.get_input_embeddings().weight.detach(), te_g.get_input_embeddings().weight.detach()
    assert float((ge - gg).abs().max()) < 1e-4
    assert torch.equal(eager.rows.slot_tokens(), graph.rows.slot_tokens())
    eager.release(); graph.release()


def _snapshot_like(graph_step, snap):
    """The graph engine's pre-prepare() snapshot, usable by the eager engine (same shapes)."""
    return {k: (v.clone() if torch.is_tensor(v) else v) for k, v in snap.items() if k != "rows"} | {
        "rows": {k: v.clone() for k, v in snap["rows"].items()}}
