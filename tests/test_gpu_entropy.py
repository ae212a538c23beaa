"""Per-token entropy from the fused lm-head pass, the entropy threshold and the entropy-masked GRPO loss on the H100: the entropy
against float64 with a per-element bound (entropy_ref.py), logp / lse bit-equal to the plain kernel, the threshold bit-equal to
torch.quantile, the loss against a float64 restatement and bit-equal to the plain / IS kernels at tau = -inf, and the trainer."""
import math

import numpy as np
import pytest
import torch

from entropy_ref import RHOS, entropy_ref, grpo_loss_ent_with_grad, threshold_cases
from gemm_ref import make_lmhead_weight, worst_ratio

pytestmark = pytest.mark.gpu
N_SMS = 132


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops as o
    return o


def _wide(M, V, K):
    """The tile width run_gemm picks (gemm_tc5.cu)."""
    return V >= 256 and K >= 512 and math.ceil(M / 128) * math.ceil(V / 256) >= 2 * N_SMS


FAMILIES = ("randn0.5", "randn3", "randn30", "spike80", "tie_two_tiles", "last_tile_max")


def _family(fam, w, M, seed):
    """bf16 h [M, K] (and the weight it goes with) whose logits z = h w^T (w ~ N(0, 9 / K): z ~ 3 |h| per unit) have the family's shape."""
    V, K = w.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    h = torch.randn(M, K, generator=g, device="cuda")
    if fam.startswith("randn"):
        return (h * float(fam[5:]) / 3).to(torch.bfloat16), w
    h = h / 3
    wf = w.float()
    if fam == "spike80":
        c = torch.randint(0, V, (M,), generator=g, device="cuda")
        gap = 80.0
    elif fam == "tie_two_tiles":
        w = w.clone()
        w[min(200, V - 1)] = w[5]                                            # two equal columns, tiles 0 and 1
        wf = w.float()
        c = torch.full((M,), 5, device="cuda")
        gap = 20.0
    else:
        c = torch.randint(((V - 1) // 128) * 128, V, (M,), generator=g, device="cuda")
        gap = 20.0
    d = wf[c]
    h = h + gap * d / (d * d).sum(1, keepdim=True)
    return h.to(torch.bfloat16), w


# V = 12296: the lm-head GEMM needs V % 8 == 0; 12296 = 96 x 128 + 8 leaves an 8-column last tile.  At K = 2048 it runs 128-wide tiles
# at M = 300 and 256-wide tiles at M = 800 (_wide).
CASES = [(151936, 2560, 300), (152000, 2560, 257), (12296, 2048, 300), (12296, 2048, 800), (1000, 2048, 129)]


@pytest.mark.parametrize("V,K,M", CASES)
def test_entropy_vs_fp64(ops, V, K, M):
    w0 = make_lmhead_weight(V, K, seed=1, device="cuda")
    worst = {}
    for i, fam in enumerate(FAMILIES):
        h, w = _family(fam, w0, M, seed=10 + i)
        scale = 0.7 if fam == "randn3" else 1.0
        tgt = torch.randint(-1, V, (M,), generator=torch.Generator(device="cuda").manual_seed(i), device="cuda")
        lp0, lse0 = ops.lmhead_logprob(h, w, tgt, scale=scale)
        lp1, lse1, ent = ops.lmhead_logprob(h, w, tgt, scale=scale, want_entropy=True)
        assert torch.equal(lp0, lp1) and torch.equal(lse0, lse1), fam        # the same bits as the plain kernel
        assert (ent >= 0).all(), fam
        ref = entropy_ref(h, w, scale, same_sign=fam in ("spike80", "tie_two_tiles", "last_tile_max"))
        worst[fam] = worst_ratio(ent, ref["H"], ref["b_H"])
    print(f"V={V} K={K} M={M} wide={_wide(M, V, K)} worst err/bound:", {k: f"{v:.3g}" for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("rho", RHOS)
def test_threshold_equals_torch_quantile(ops, rho):
    for name, x, m in threshold_cases():
        x, m = x.cuda(), m.cuda()
        tau = ops.entropy_threshold(x, m, 1.0 - rho)
        valid = x[m != 0]
        want = torch.quantile(valid, 1.0 - rho).reshape(1) if valid.numel() else torch.full((1,), math.inf, device="cuda")
        assert tau.view(torch.int32).item() == want.view(torch.int32).item(), (name, rho, tau.item(), want.item())


def _loss_case(B, C, seed):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, C, generator=g) * 3
    old = lp + torch.randn(B, C, generator=g) * 0.2
    ref = lp + torch.randn(B, C, generator=g) * 0.2
    samp = lp + torch.randn(B, C, generator=g) * 0.5
    ent = torch.rand(B, C, generator=g) * 5
    adv = torch.randn(B, generator=g)
    mask = (torch.arange(C)[None, :] < torch.randint(0, C + 1, (B, 1), generator=g)).int()
    return [t.cuda() for t in (lp, old, ref, samp, ent, adv, mask)]


@pytest.mark.parametrize("B,C", [(16, 300), (48, 97)])
@pytest.mark.parametrize("beta", [0.0, 0.04])
@pytest.mark.parametrize("is_on", [False, True])
def test_loss_kernel_vs_fp64(ops, B, C, beta, is_on):
    lp, old, ref, samp, ent, adv, mask = _loss_case(B, C, seed=B + C)
    tau = ops.entropy_threshold(ent, mask, 0.8)
    rl = samp if is_on else None
    out3, stats, ent_sum, dlp = ops.grpo_loss_ent_raw(lp, old, ref if beta else None, rl, adv, mask, ent, tau, beta, 0.2, 0.28, 2.0)
    want, kl, clip, es, grad = grpo_loss_ent_with_grad(lp, old, ref if beta else None, rl, adv, mask, ent, tau.item(), beta, 0.2, 0.28, 2.0)
    torch.testing.assert_close(out3[0].double(), want, rtol=2e-5, atol=1e-7)
    torch.testing.assert_close(out3[2].double(), clip, rtol=2e-5, atol=1e-7)
    if beta:
        torch.testing.assert_close(out3[1].double(), kl, rtol=2e-5, atol=1e-7)
    torch.testing.assert_close(ent_sum[0].double(), es, rtol=2e-5, atol=1e-5)
    torch.testing.assert_close(dlp.double(), grad, rtol=2e-5, atol=1e-9)
    kept = ((ent >= tau) & (mask != 0)).sum().item()
    assert 0 < kept < mask.sum().item()
    # tau = -inf: the plain / IS kernel, bit for bit
    ninf = torch.full((1,), -math.inf, device="cuda")
    o1, s1, _, d1 = ops.grpo_loss_ent_raw(lp, old, ref if beta else None, rl, adv, mask, ent, ninf, beta, 0.2, 0.28, 2.0)
    if is_on:
        o0, s0, d0 = ops.grpo_loss_is_raw(lp, old, ref if beta else None, samp, adv, mask, beta, 0.2, 0.28, 2.0)
        assert torch.equal(s0, s1)
    else:
        o0, d0 = ops.grpo_loss_raw(lp, old, ref if beta else None, adv, mask, beta, 0.2, 0.28)
    assert torch.equal(o0, o1) and torch.equal(d0, d1)


# ------------------------------------------------------------------------------------------------------------------- trainer
def _token_reward(completion_ids, **kw):
    return (completion_ids % 7 == 0).float().sum(1) - 0.1 * (completion_ids % 5 == 0).float().sum(1)


def _trainer(rho=1.0, log_entropy=False, mu=1, share=False, beta=0.04, micro_rows=None, tis=False, fp8=False, dropout=False, ga=1,
             live_b=True, seed=21):
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config("tiny"), dna_config("tiny")
    oracle = build_oracle(tc, dc, seed=seed)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14, same_prompt=True)
    m = DNALLMModel.from_oracle(oracle)
    cfg = DNALLMGRPOConfig(num_generations=4, max_completion_length=8, per_device_train_batch_size=4, learning_rate=1e-2, lora_r=16,
                           lora_alpha=32.0, num_iterations=mu, beta=beta, share_prompt_prefix=share, micro_rows=micro_rows,
                           fp8_rollout=fp8, rollout_is_correction=tis, apply_lora_dropout=dropout, lora_dropout=0.1,
                           gradient_accumulation_steps=ga, top_entropy_quantile=rho, log_entropy=log_entropy)
    tr = DNALLMGRPOTrainer(m, [_token_reward], cfg)
    if live_b:
        with torch.no_grad():
            g = torch.Generator().manual_seed(5)
            for p in m._lora.params[1::2]:
                p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device))
        m.sync_adapters(rollout=True)
    return tr, m, batch, oracle


def _run(tr, m, inputs, **args):
    for k, v in args.items():
        setattr(tr.args, k, v)
    tr._step, tr.global_step = 0, 0
    tr._metrics.clear()
    m.zero_grad_buffers()
    loss = tr.compute_loss(m, inputs)
    grads = [m._lora.flat_grad.clone(), m._proj_grad_w.clone(), m._proj_grad_b.clone()]
    return loss.clone(), grads, {k: [float(x) for x in v] for k, v in tr._metrics.items()}


def _inputs(tr, m, batch):
    inputs = tr._generate_and_score_completions(batch, m, uniforms=torch.rand(8, 4, generator=torch.Generator().manual_seed(0)).cuda())
    inputs["advantages"] = torch.tensor([1.0, -0.5, 0.3, -0.8], device="cuda")
    return inputs


def test_log_entropy_leaves_loss_and_gradients_bit_identical():
    tr, m, batch, _ = _trainer()
    inputs = _inputs(tr, m, batch)
    l0, g0, met0 = _run(tr, m, inputs, log_entropy=False)
    l1, g1, met1 = _run(tr, m, inputs, log_entropy=True)
    assert torch.equal(l0, l1) and all(torch.equal(a, b) for a, b in zip(g0, g1))
    assert "entropy" not in met0 and met1["entropy"][0] > 0 and "entropy/threshold" not in met1


def test_prepass_equals_one_chunk():
    """micro_rows = 2 (two chunks: the no-grad pre-pass decides the mask) against one chunk (the loss pass's own entropies): the same
    threshold, mask and loss; the gradients differ only in the fp32 order of the chunk sums."""
    tr, m, batch, _ = _trainer(rho=0.2)
    inputs = _inputs(tr, m, batch)
    l1, g1, met1 = _run(tr, m, inputs, micro_rows=4)
    l2, g2, met2 = _run(tr, m, inputs, micro_rows=2)
    assert met1["entropy/threshold"] == met2["entropy/threshold"]
    assert abs(met1["entropy"][0] - met2["entropy"][0]) <= 1e-6 * met1["entropy"][0]
    torch.testing.assert_close(l1, l2, rtol=1e-6, atol=1e-7)
    for a, b in zip(g1, g2):
        assert torch.any(a != 0)
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-6 * a.abs().max().item())


def test_prepass_under_lora_dropout():
    """Two chunks under LoRA dropout: the pre-pass reproduces the loss pass's dropout masks, so its entropies are the loss pass's bit for
    bit (compute_loss raises otherwise)."""
    tr, m, batch, _ = _trainer(rho=0.2, dropout=True)
    inputs = _inputs(tr, m, batch)
    loss, grads, met = _run(tr, m, inputs, micro_rows=2)
    assert torch.isfinite(loss) and met["entropy"][0] > 0


def test_training_step_vs_fp32_oracle():
    """rho = 0.2 with LoRA B = 0 (policy = the oracle's base model): the trainer's loss against TRL's formula on the fp32 oracle's
    logits.  Tokens whose oracle entropy lies within the largest |H_kernel - H_oracle| of tau are at risk: they take the kernel's
    decision in the oracle's loss."""
    from oracle import grpo as og
    tr, m, batch, oracle = _trainer(rho=0.2, live_b=False)
    inputs = _inputs(tr, m, batch)
    comp, cmask = inputs["completion_ids"], inputs["completion_mask"]
    C = comp.shape[1]
    ids = torch.cat([inputs["prompt_ids"], comp], 1)
    mask = torch.cat([inputs["prompt_mask"], cmask.to(inputs["prompt_mask"].dtype)], 1)
    mm = inputs["multimodal_inputs"]
    _, ent_k = tr._get_per_token_logps_and_entropies(m, ids, mask, C, **mm)
    loss, _, met = _run(tr, m, inputs)
    tau_k = met["entropy/threshold"][0]
    with torch.no_grad():
        logits = oracle(input_ids=ids.cpu(), attention_mask=mask.cpu(), dna_tokenized={k: v.cpu() for k, v in mm["dna_tokenized"].items()},
                        batch_idx_map=mm["batch_idx_map"]).logits[:, -C - 1:-1].float()
    lsm = torch.log_softmax(logits, -1)
    ent_o = -(lsm.exp() * lsm).sum(-1)
    lp_o = lsm.gather(-1, comp.cpu()[..., None])[..., 0]
    valid = cmask.cpu() != 0
    tau_o = torch.quantile(ent_o[valid], 0.8).item()
    margin = (ent_k.cpu() - ent_o)[valid].abs().max().item()
    keep_o = (ent_o >= tau_o) & valid
    keep_k = (ent_k.cpu() >= tau_k) & valid
    risk = ((ent_o - tau_o).abs() <= margin + abs(tau_k - tau_o)) & valid
    keep = torch.where(risk, keep_k, keep_o)
    n_masked = (valid & ~keep).sum().item()
    assert n_masked >= 0.1 * valid.sum().item()
    print(f"valid {valid.sum().item()}, masked {n_masked}, at risk {risk.sum().item()}, entropy margin {margin:.3g}, "
          f"tau kernel {tau_k:.6g} oracle {tau_o:.6g}")
    want, _, _, _, _ = grpo_loss_ent_with_grad(lp_o, None, lp_o, None, inputs["advantages"].cpu(), cmask.cpu(), keep.float(), 0.5,
                                               0.04, 0.2, 0.2)
    assert abs(loss.item() - want.item()) < 5e-3


@pytest.mark.parametrize("combo", ["share", "mu2", "beta0", "tis", "fp8", "dropout", "ga2"])
def test_every_combination_runs_a_step(combo):
    kw = dict(share=dict(share=True), mu2=dict(mu=2), beta0=dict(beta=0.0), tis=dict(tis=True), fp8=dict(fp8=True),
              dropout=dict(dropout=True, micro_rows=2), ga2=dict(ga=2))[combo]
    tr, m, batch, _ = _trainer(rho=0.2, **kw)
    for _ in range(2):
        assert torch.isfinite(tr.training_step(batch))
    met = tr.log_metrics()
    assert met["entropy"] > 0 and math.isfinite(met["entropy/threshold"])
