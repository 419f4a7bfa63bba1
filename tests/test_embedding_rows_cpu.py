"""Jointly trained embedding rows without a GPU: the three C entry points are declared, exported and
refuse bad arguments before any CUDA call; the oracle's `continue_inversion` loop
(oracle/joint_ref.py, mode "table") reproduces the reference's real `perform_tuning` run with the
token-embedding table in the optimizer (tests/golden/pti_continue_inversion.pt)."""
import ctypes
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("lb_embed_rows_scatter", "lb_embed_rows_write_back", "lb_embed_rows_flush")


def test_embedding_row_entry_points_are_declared_and_exported():
    from lora_b200 import _C
    header = open(os.path.join(ROOT, "include", "lora_b200.h")).read()
    lib = ctypes.CDLL(_C.LIB_PATH)
    for n in NAMES:
        assert f"int {n}(" in header
        assert hasattr(lib, n) and n in _C.EXPORTED


def test_embedding_row_entry_points_validate_without_gpu():
    from lora_b200 import _C
    L = _C.lib
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.c_void_p((ctypes.addressof(buf) + 255) & ~255)
    SHAPE, DTYPE = -1, -3
    BF16, F32 = _C.LB_BF16, _C.LB_F32

    def scatter(**kw):
        a = dict(ids=p, grad=p, gdt=F32, n=77, D=48, V=1000, slot_of=p, slot_tok=p, cap=8, state=p, table=p,
                 tdt=F32, decay=p, master=p, sgrad=p)
        a.update(kw)
        return L.lb_embed_rows_scatter(a["ids"], a["grad"], a["gdt"], a["n"], a["D"], a["V"], a["slot_of"],
                                       a["slot_tok"], a["cap"], a["state"], a["table"], a["tdt"], a["decay"],
                                       a["master"], a["sgrad"], None)

    for k in ("ids", "grad", "slot_of", "slot_tok", "state", "table", "decay", "master", "sgrad"):
        assert scatter(**{k: None}) == SHAPE, k
    assert scatter(D=0) == SHAPE and scatter(V=0) == SHAPE and scatter(cap=0) == SHAPE
    assert scatter(n=0) == SHAPE and scatter(n=2049) == SHAPE      # B*S above the launch's bookkeeping
    assert scatter(gdt=7) == DTYPE and scatter(tdt=-1) == DTYPE

    def write_back(**kw):
        a = dict(master=p, slot_tok=p, cap=8, state=p, n_write=-1, table=p, tdt=BF16, D=48, V=1000, decay=p,
                 lr=p, lr_index=2, wd=1e-3)
        a.update(kw)
        return L.lb_embed_rows_write_back(a["master"], a["slot_tok"], a["cap"], a["state"], a["n_write"],
                                          a["table"], a["tdt"], a["D"], a["V"], a["decay"], a["lr"],
                                          a["lr_index"], a["wd"], None)

    for k in ("master", "slot_tok", "state", "table"):
        assert write_back(**{k: None}) == SHAPE, k
    assert write_back(D=0) == SHAPE and write_back(V=0) == SHAPE and write_back(cap=0) == SHAPE
    assert write_back(lr_index=-1) == SHAPE
    assert write_back(decay=None) == SHAPE and write_back(lr=None) == SHAPE   # both or neither
    assert write_back(tdt=5) == DTYPE

    def flush(**kw):
        a = dict(table=p, tdt=F32, V=1000, D=48, slot_of=p, decay=p, state=p)
        a.update(kw)
        return L.lb_embed_rows_flush(a["table"], a["tdt"], a["V"], a["D"], a["slot_of"], a["decay"], a["state"], None)

    for k in ("table", "slot_of", "decay", "state"):
        assert flush(**{k: None}) == SHAPE, k
    assert flush(V=0) == SHAPE and flush(D=-3) == SHAPE
    assert flush(tdt=3) == DTYPE


def test_joint_oracle_matches_reference_continue_inversion_golden():
    """oracle/joint_ref.py (mode "table": scheduler first, t < 0.8 T, backward, clip over UNet + text
    encoder, AdamW over [unet LoRA, dense table, text LoRA]) against 3 iterations of the reference's
    real `perform_tuning` built with continue_inversion=True (golden from
    scripts/make_golden.py::gen_continue_inversion): per-step loss and lrs, whole table after every step."""
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.ddpm import DDPMNoiser
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from oracle.joint_ref import RefJointStep
    from oracle.ref_modules import ref_inject
    G = torch.load(os.path.join(ROOT, "tests", "golden", "pti_continue_inversion.pt"))
    torch.manual_seed(G["model_seed"])
    unet = UNet2DConditionModel(UNetConfig.tiny())
    text = build_text_encoder(tiny=True)
    table = text.get_input_embeddings().weight
    assert torch.equal(table.detach(), G["table0"]) and tuple(table.shape) == (1000, 48)
    us = ref_inject(unet, {"CrossAttention", "Attention", "GEGLU"}, r=4)
    ts = ref_inject(text, {"CLIPAttention"}, r=4)
    assert len(us) == G["n_unet_sites"]
    gg = torch.Generator().manual_seed(G["factor_seed"])
    for s in us + ts:
        s.down.data.normal_(0, 0.25, generator=gg)
        s.up.data.normal_(0, 0.05, generator=gg)
    lr, lr_emb, lr_text = G["lrs0"]
    ref = RefJointStep(unet, text, DDPMNoiser(device="cpu"), us, ts, "table", lr=lr, lr_text=lr_text,
                       lr_embedding=lr_emb, lr_lambda=lambda k: max(0.0, 1.0 - k / 6),
                       weight_decay=G["weight_decay"], t_multiplier=0.8)
    torch.manual_seed(G["step_seed"])
    for st, batch in zip(G["steps"], G["batches"]):
        loss = ref.step(batch["pixel_values"], batch["input_ids"])
        assert ref.lrs() == st["lrs"]
        assert abs(float(loss) - st["loss"]) <= 5e-6 * abs(st["loss"]), (float(loss), st["loss"])
        assert torch.allclose(ref.table.detach(), st["table_after"], rtol=0, atol=2e-7)
    # every row moved (weight decay), the rows of the batches' tokens by far the most
    seen = torch.unique(torch.cat([b["input_ids"].reshape(-1) for b in G["batches"]]))
    moved = (G["steps"][-1]["table_after"] - G["table0"]).abs().amax(dim=1)
    unseen = torch.ones(1000, dtype=torch.bool)
    unseen[seen] = False
    assert float(moved[unseen].min()) > 0 and float(moved[seen].min()) > 100 * float(moved[unseen].max())
