"""Per-image LoRA coefficients without a GPU: the three _ps entry points are declared, typed and
exported and refuse bad tables before any CUDA call; the coefficient tables are fl32(fl32(s) * fl32(d))
with defaults from each site's scale and selector; LoRAManager.diag_rows is what tune() sets; and the
samplers and per_sample_lora refuse bad arguments."""
import ctypes
import types

import pytest
import torch

from test_cabi import _declared

PS = ("lb_lora_linear_fwd_ps", "lb_lora_linear_fwd_grouped_ps", "lb_lora_conv2d_fwd_ps",
      "lb_lora_linear_fwd_split_k", "lb_lora_conv2d_fwd_split_k")


def test_entry_points_are_declared_typed_and_exported():
    from lora_b200 import _C
    names = _declared()
    for n in PS:
        assert n in names and n in _C.EXPORTED
        fn = getattr(_C.lib, n)
        assert fn.argtypes is not None and fn.restype is ctypes.c_int
    assert _C.lib.lb_abi_version() == 7


def test_entry_points_refuse_bad_tables_without_gpu():
    from lora_b200 import _C
    L = _C.lib
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.c_void_p((ctypes.addressof(buf) + 255) & ~255)
    lin = lambda coef, ld, rps, S, r=4, rp=16, dt=0: L.lb_lora_linear_fwd_ps(
        p, p, None, p, p, 4, 1, coef, ld, rps, S, p, 8, 64, 64, r, rp, dt, dt, None)
    assert lin(None, 4, 1, 1) == -1          # no table
    assert lin(p, 3, 1, 1) == -1             # row pitch below the rank
    assert lin(p, 4, 0, 1) == -1             # rows_per_sample 0
    assert lin(p, 4, 1, 0) == -1             # no samples
    assert lin(p, 17, 1, 1, r=17) == -2      # rank beyond its pad
    assert lin(p, 4, 1, 1, dt=2) == -3       # fp32 operands
    conv = lambda coef, ld, rps, S, kh=3: L.lb_lora_conv2d_fwd_ps(
        p, p, None, p, p, 4, 1, coef, ld, rps, S, p, 1, 8, 8, 64, 64, kh, kh, kh // 2, kh // 2, 4, 16, 0, 0, None)
    assert conv(None, 4, 64, 1) == -1
    assert conv(p, 2, 64, 1) == -1
    assert conv(p, 4, 64, 1, kh=5) == -1     # geometry checks still apply
    arr = lambda ty, *v: (ty * len(v))(*v)
    VP, I, LL = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    grouped = lambda coef, ld: L.lb_lora_linear_fwd_grouped_ps(
        1, arr(VP, p.value), arr(VP, p.value), None, arr(VP, p.value), arr(VP, p.value), arr(LL, 4), arr(LL, 1),
        coef, ld, arr(I, 1), arr(I, 1), arr(VP, p.value), arr(I, 8), arr(I, 64), arr(I, 64), arr(I, 4), 0, 0, None)
    assert grouped(None, arr(I, 4)) == -1
    assert grouped(arr(VP, p.value), arr(I, 2)) == -1
    assert grouped(arr(VP, None), arr(I, 4)) == -1
    # the planner queries refuse bad shapes and rank pads
    assert L.lb_lora_linear_fwd_split_k(0, 64, 64, 16) == -1
    assert L.lb_lora_linear_fwd_split_k(8, 64, 64, 24) == -1
    assert L.lb_lora_conv2d_fwd_split_k(1, 8, 8, 64, 64, 3, 3, 48) == -1
    assert L.lb_lora_conv2d_fwd_split_k(0, 8, 8, 64, 64, 3, 3, 16) == -1


def _sites(r=4, n=3):
    import lora_b200 as L
    torch.manual_seed(0)
    return [L.LoraInjectedLinear(16, 16, r=r, dropout_p=0.0, scale=0.1 * (i + 1)) for i in range(n)]


def test_table_entries_are_fp32_products_with_module_defaults():
    from lora_b200 import per_sample
    sites = _sites()
    sites[1].set_selector_from_diag(torch.tensor([0.3, 1.0, -2.0, 1.7]))
    S = 3
    scales = [0.1, 1.0 / 3.0, 7.25]
    diag = torch.tensor([[0.7, 1.1, 0.0, 3.3], [1.0, 1.0, 1.0, 1.0], [0.2, 0.9, 1e-3, 5.0]], dtype=torch.float64)
    for sc, dg in ((scales, diag), (None, diag), (scales, None), (None, None), (0.6, diag[0])):
        s32, d32 = per_sample.check_args(sites, sc, dg, S)
        flat = per_sample.host_table(sites, s32, d32, S)
        assert flat.dtype == torch.float32 and flat.numel() == S * 4 * len(sites)
        for m, v in zip(sites, per_sample.table_views(flat, sites, S)):
            s = torch.tensor(float(m.scale) if sc is None else sc, dtype=torch.float32).expand(S)
            if dg is None:
                d = m._selector_diag()
                d = torch.ones(4) if d is None else d
                d = d.float().expand(S, 4)
            else:
                d = dg.float().expand(S, 4)
            assert torch.equal(v, s[:, None] * d)
            for b in range(S):   # one element at a time: fl32(fl32(s_b) * fl32(d_bj))
                for j in range(4):
                    want = torch.tensor(float(s[b]), dtype=torch.float32) * torch.tensor(float(d[b, j]),
                                                                                         dtype=torch.float32)
                    assert v[b, j].item() == want.item()


def test_uniform_rows_equal_the_scalar_coefficients():
    from lora_b200 import per_sample
    m = _sites(n=1)[0]
    m.scale = 0.7
    m.set_selector_from_diag(torch.tensor([0.25, 1.5, 3.0, 0.1]))
    t = per_sample.site_rows(m, None, None, 5)
    # the kernel's scalar path: fl32(scale) * diag[j] in fp32
    want = torch.tensor(0.7, dtype=torch.float32) * m._selector_diag()
    assert all(torch.equal(t[b], want) for b in range(5))


def test_diag_rows_are_what_tune_sets():
    import lora_b200 as L
    sites = _sites(r=5, n=2)
    model = torch.nn.Sequential(*sites)
    mgr = L.LoRAManager.__new__(L.LoRAManager)
    mgr.ranklist, mgr.pipe = [2, 3], types.SimpleNamespace(unet=model)
    mixes = [[1.0, 0.0], [0.3, 0.9], [2.0, 0.5]]
    rows = mgr.diag_rows(mixes)
    assert rows.shape == (3, 5) and rows.dtype == torch.float32
    for b, mix in enumerate(mixes):
        mgr.tune(mix)
        for m in sites:
            assert torch.equal(rows[b], m._selector_diag())
    with pytest.raises(AssertionError):
        mgr.diag_rows([[1.0]])


def test_per_sample_lora_argument_validation():
    import lora_b200 as L
    sites = _sites()
    model = torch.nn.Sequential(*sites)
    with pytest.raises(ValueError, match="samples"):
        with L.per_sample_lora(model, scale=0.5):
            pass
    with pytest.raises(ValueError, match="one per image"):
        with L.per_sample_lora(model, scale=[0.5, 1.0], samples=3):
            pass
    with pytest.raises(ValueError, match="rank 4"):
        with L.per_sample_lora(model, diag=torch.ones(2, 5)):
            pass
    with pytest.raises(ValueError, match="no LoRA sites"):
        with L.per_sample_lora(torch.nn.Linear(4, 4), scale=[1.0]):
            pass
    mixed = torch.nn.Sequential(_sites(r=4, n=1)[0], _sites(r=2, n=1)[0])
    with pytest.raises(ValueError, match="one rank"):
        with L.per_sample_lora(mixed, diag=torch.ones(2, 4)):
            pass
    # a good call binds every site on entry and unbinds on exit (CPU tables for CPU sites)
    with L.per_sample_lora(model, scale=[0.5, 1.0]):
        assert all(m._lb.ps is not None and m._lb.ps[1] == 2 and m._lb.ps[0].shape == (2, 4) for m in sites)
    assert all(m._lb.ps is None for m in sites)


def _tiny_sampler():
    from lora_b200.host.clip import build_text_encoder
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.host.vae import AutoencoderKL, VAEConfig
    from lora_b200.sample import LoraSampler, SamplerConfig
    import lora_b200 as L
    unet, text = UNet2DConditionModel(UNetConfig.tiny()), build_text_encoder(tiny=True)
    L.inject_trainable_lora(unet, r=4)
    vae = AutoencoderKL(VAEConfig.tiny(), with_decoder=True)
    return LoraSampler(unet, text, vae, SamplerConfig(max_steps=4, num_inference_steps=4, external_noise=True),
                       latent_shape=(2, 4, 8, 8), device="cpu")


def test_sampler_per_sample_argument_validation():
    s = _tiny_sampler()
    ids = torch.zeros(2, 77, dtype=torch.long)
    bad = [
        (dict(lora_scale={"unet": [1.0, 2.0, 3.0]}), "one per image"),
        (dict(lora_scale={"vae": 1.0}), "unknown model"),
        (dict(lora_scale=[1.0, 2.0]), "model names"),
        (dict(lora_diag={"unet": torch.ones(2, 3)}), "rank 4"),
        (dict(lora_diag={"unet": torch.ones(3, 4)}), "one row per image"),
        (dict(lora_scale={"text_encoder": 0.5}), "no LoRA sites"),     # the text encoder has none here
        (dict(shared_noise=True), "external_noise"),
    ]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            s.sample(ids, ids, **kw)
    assert s.captures == 0
    plan = s._per_sample_plan({"unet": [0.5, 1.0]}, {"unet": torch.ones(4)})
    assert set(plan) == {"unet"} and plan["unet"][0].tolist() == [0.5, 1.0] and plan["unet"][1].shape == (2, 4)
    assert s._per_sample_plan(None, None) is None


def test_per_sample_fingerprint_leaves_scale_and_selector_out():
    import lora_b200 as L
    s = _tiny_sampler()
    full, struct = s._fingerprint_now(), s._fingerprint_now(structural=True)
    L.tune_lora_scale(s.unet, 0.3)
    L.set_lora_diag(s.unet, torch.tensor([1.0, 0.0, 0.5, 2.0]))
    assert s._fingerprint_now() != full and s._fingerprint_now(structural=True) == struct
    assert s._key(2, "single-step", False) + ("per_sample",) != s._key(2, "single-step", False)


def test_xl_sampler_takes_text_encoder_2_by_its_save_safeloras_name():
    from lora_b200.sample import LoraXLSampler
    names = LoraXLSampler._model_names(types.SimpleNamespace(unet=1, text_encoder=2, text_encoder_2=3))
    assert names == {"unet": 1, "text_encoder": 2, "text_encoder_2": 3}
