"""The data-parallel gradient scatter without a GPU: lb_embed_rows_scatter_dp is declared, exported and
refuses bad arguments (null pointers, world < 1, rank >= world, more than 2048 tokens over all ranks,
half a handshake) before any CUDA call; LoraEmbeddingStep's token limit is the same number."""
import ctypes
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "lb_embed_rows_scatter_dp"


def test_dp_scatter_is_declared_and_exported():
    from lora_b200 import _C
    header = open(os.path.join(ROOT, "include", "lora_b200.h")).read()
    lib = ctypes.CDLL(_C.LIB_PATH)
    assert f"int {NAME}(" in header
    assert hasattr(lib, NAME) and NAME in _C.EXPORTED


def test_dp_scatter_validates_without_gpu():
    from lora_b200 import _C
    from lora_b200.embed_rows import MAX_SCATTER_TOKENS
    assert MAX_SCATTER_TOKENS == 2048
    L = _C.lib
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.c_void_p((ctypes.addressof(buf) + 255) & ~255)
    SHAPE, DTYPE = -1, -3
    F32 = _C.LB_F32
    VP = ctypes.c_void_p * 16

    def scatter(world=2, rank=0, n=77, ids=None, flags=None, epoch=None, **kw):
        ids = VP(*([p.value] * 16)) if ids is None else ids
        a = dict(grad=p, gdt=F32, D=48, V=1000, slot_of=p, slot_tok=p, cap=8, state=p, table=p, tdt=F32, decay=p,
                 master=p, sgrad=p)
        a.update(kw)
        return L.lb_embed_rows_scatter_dp(ids, world, rank, n, a["grad"], a["gdt"], a["D"], a["V"], a["slot_of"],
                                          a["slot_tok"], a["cap"], a["state"], a["table"], a["tdt"], a["decay"],
                                          a["master"], a["sgrad"], flags, epoch, None)

    for k in ("grad", "slot_of", "slot_tok", "state", "table", "decay", "master", "sgrad"):
        assert scatter(**{k: None}) == SHAPE, k
    null_ids = ctypes.c_void_p * 2
    assert L.lb_embed_rows_scatter_dp(None, 1, 0, 77, p, F32, 48, 1000, p, p, 8, p, p, F32, p, p, p, None, None,
                                      None) == SHAPE
    assert scatter(ids=null_ids(p.value, None)) == SHAPE            # rank 1's ids missing
    assert scatter(world=0) == SHAPE and scatter(world=-1) == SHAPE and scatter(world=17) == SHAPE
    assert scatter(rank=2) == SHAPE and scatter(rank=-1) == SHAPE and scatter(world=4, rank=4) == SHAPE
    assert scatter(n=0) == SHAPE
    # the union of all ranks' tokens is what the launch's bookkeeping holds
    assert scatter(world=2, n=1025) == SHAPE and scatter(world=8, n=257) == SHAPE
    assert scatter(world=8, n=2 * 77, D=0) == SHAPE               # 8 ranks x bs 2 x 77 fits; D=0 is refused
    assert scatter(D=0) == SHAPE and scatter(V=0) == SHAPE and scatter(cap=0) == SHAPE
    assert scatter(gdt=7) == DTYPE and scatter(tdt=-1) == DTYPE
    # the handshake needs both the flags and the epoch, and every rank's flag
    assert scatter(flags=VP(*([p.value] * 16))) == SHAPE
    assert scatter(epoch=p) == SHAPE
    assert scatter(flags=null_ids(p.value, None), epoch=p) == SHAPE


def test_embedding_step_checks_the_token_limit_at_construction():
    """Outside torch.distributed the limit is B * S <= 2048: refused before any model or CUDA work."""
    import pytest
    import torch
    from lora_b200._C import LoraB200Error
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.train import LoraEmbeddingStep, StepConfig
    text = build_text_encoder(tiny=True)
    with pytest.raises(LoraB200Error, match="2048"):
        LoraEmbeddingStep(torch.nn.Module(), text, [998], StepConfig(), lr_embedding=1e-4,
                          latent_shape=(27, 4, 8, 8), seq_len=77)
