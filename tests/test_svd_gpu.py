"""GPU parity of the batched truncated SVD (csrc/svd.cu, lora_b200/svd.py) against the oracle's
exact SVD (oracle/svd_ref.py, restating cli_svd.py:24-92), on the sign-invariant quantities:
singular values, the rank-r product before clamping, orthonormality of the right factor, and the
clamp rule. Inputs: dW = lowrank(8) * 0.02 + noise * 1e-3, fp16 weights."""
import pytest
import torch

from oracle import svd_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def make_pairs(N, K, batch, true_rank=8, dtype=torch.float16, seed=0):
    g = torch.Generator().manual_seed(seed)
    Wb, Wt = [], []
    for _ in range(batch):
        base = torch.randn(N, K, generator=g) * 0.05
        # decaying spectrum so that the top-r triplets are well separated
        s = torch.tensor([1.0 / (1 + 0.35 * i) for i in range(true_rank)])
        low = (torch.randn(N, true_rank, generator=g) * s) @ torch.randn(true_rank, K, generator=g) * 0.02 / (K ** 0.5) * 8
        noise = torch.randn(N, K, generator=g) * 1e-3
        Wb.append(base.to(dtype))
        Wt.append((base + low + noise).to(dtype))
    return Wb, Wt


@pytest.mark.parametrize("N,K,batch,rank", [(320, 320, 6, 8), (2560, 320, 2, 8), (320, 768, 3, 4),
                                            (1280, 1280, 2, 8), (768, 768, 4, 16), (10240, 1280, 1, 8),
                                            (96, 200, 2, 1)])
def test_batched_svd_matches_exact_svd(N, K, batch, rank):
    from lora_b200.svd import svd_lowrank_batched
    # the planted spectrum must be at least as wide as the requested rank (below it, singular
    # vectors of the isotropic noise floor are not unique)
    Wb, Wt = make_pairs(N, K, batch, true_rank=max(8, rank), seed=N + K)
    up, down, sigma = svd_lowrank_batched([w.to(DEV) for w in Wt], [w.to(DEV) for w in Wb], rank)
    torch.cuda.synchronize()
    for b in range(batch):
        resid = (Wt[b].float() - Wb[b].float())           # what the reference forms (cli_svd.py:31-33)
        U, S, Vh = torch.linalg.svd(resid.double(), full_matrices=False)
        assert rel(sigma[b, :rank], S[:rank]) < 2e-3
        exact = (U[:, :rank] * S[:rank]) @ Vh[:rank]
        ours = up[b].double().cpu() @ down[b].double().cpu()
        assert rel(ours, exact) < 5e-3
        # Eckart-Young: our rank-r residual is within 0.1% of the optimum
        opt = (resid.double() - exact).norm()
        got = (resid.double() - ours).norm()
        assert float(got) <= float(opt) * 1.001 + 1e-12
        gram = down[b].double().cpu() @ down[b].double().cpu().T
        assert rel(gram, torch.eye(rank, dtype=torch.float64)) < 2e-3


def test_exactly_low_rank_delta_is_handled():
    """dW of exact rank 3 (a merged LoRA), asked for rank 8: the 5 surplus triplets are zero, no NaN."""
    from lora_b200.svd import svd_lowrank_batched
    g = torch.Generator().manual_seed(0)
    base = (torch.randn(640, 320, generator=g) * 0.05)
    low = torch.randn(640, 3, generator=g) @ torch.randn(3, 320, generator=g) * 0.01
    up, down, sigma = svd_lowrank_batched([(base + low).to(DEV)], [base.to(DEV)], 8)
    torch.cuda.synchronize()
    assert torch.isfinite(up).all() and torch.isfinite(down).all() and torch.isfinite(sigma).all()
    S = torch.linalg.svdvals(low.double())
    assert rel(sigma[0, :3], S[:3]) < 1e-3
    assert float(sigma[0, 3:8].max()) < 1e-4 * float(S[0])
    assert rel(up[0].double().cpu() @ down[0].double().cpu(), low) < 1e-3


def test_overwrite_base_matches_oracle_on_tiny_models():
    import copy
    import lora_b200 as L
    from lora_b200.host.unet_sd15 import UNet2DConditionModel, UNetConfig
    from lora_b200.svd import overwrite_base
    torch.manual_seed(0)
    base = UNet2DConditionModel(UNetConfig.tiny()).to(DEV).half()
    tuned = copy.deepcopy(base)
    g = torch.Generator(device=DEV).manual_seed(1)
    for p in tuned.parameters():
        if p.dim() >= 2:
            n, k = p.shape[0], p[0].numel()
            low = (torch.randn(n, 4, device=DEV, generator=g) @ torch.randn(4, k, device=DEV, generator=g)) * 0.01
            p.data.add_(low.reshape(p.shape).half())
    L.inject_trainable_lora_extended(base, r=4)
    L.inject_trainable_lora_extended(tuned, r=4)
    overwrite_base(base, tuned, rank=4, clamp_quantile=0.99)
    torch.cuda.synchronize()
    sb = [m for m in base.modules() if type(m).__name__.startswith("LoraInjected")]
    stn = [m for m in tuned.modules() if type(m).__name__.startswith("LoraInjected")]
    assert len(sb) > 10
    for a, t in zip(sb, stn):
        wa = (a.linear if hasattr(a, "linear") else a.conv).weight.data
        wt = (t.linear if hasattr(t, "linear") else t.conv).weight.data
        up_o, down_o, S, hi = svd_ref.svd_distill_pair(wa.cpu(), wt.cpu(), 4, 0.99)
        assert a.lora_up.weight.shape == up_o.shape and a.lora_down.weight.shape == down_o.shape
        assert a.lora_up.weight.dtype == torch.float16
        ours = a.lora_up.weight.data.float().flatten(1).cpu() @ a.lora_down.weight.data.float().flatten(1).cpu()
        # The reference's threshold `hi` is a quantile over SIGNED factor entries, hence depends on the
        # (arbitrary) sign of each singular pair. Sign-invariant statement: clamping the
        # exact factors at OUR threshold reproduces our clamped product.
        u2, d2, hi_ours = svd_ref.clamp_rule(a.lora_up.weight.data.float().cpu(), a.lora_down.weight.data.float().cpu(), 0.99)
        hi_eff = float(max(a.lora_up.weight.data.abs().max(), a.lora_down.weight.data.abs().max()))
        resid = (wt.float() - wa.float()).flatten(1).cpu()
        U, S_, Vh = torch.linalg.svd(resid, full_matrices=False)
        Ue, Ve = (U[:, :4] * S_[:4]).clamp(-hi_eff, hi_eff), Vh[:4].clamp(-hi_eff, hi_eff)
        assert rel(ours, Ue @ Ve) < 3e-2
        # the reference's own threshold differs only through the sign convention (same order of magnitude;
        # on these 32..128-wide toy matrices the 0.99 quantile is a noisy statistic)
        assert 0.3 * hi < hi_eff < 3.0 * hi
