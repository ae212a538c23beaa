"""The GRPO objectives of later TRL releases on the GPU: br_grpo_objective_fwd_bwd against the float64 restatement in
grpo_objective_ref.py, its identities (the existing loss kernels' bits at the defaults, sequence = token level at mu = 1), the advantage
and truncated-mask kernels, and training steps against autograd of the contract on the fp32 oracle."""
import math

import pytest
import torch

from grpo_objective_ref import advantages as adv_ref, objective, objective_with_grad, token_terms, truncated_mask

pytestmark = pytest.mark.gpu

LOSS_TYPES = ["grpo", "bnpo", "dr_grpo", "dapo"]
SHAPES = [(b, c) for b in (1, 3, 8, 33) for c in (1, 7, 512, 4096)]
MAXLEN, WORLD = 4500, 2                      # dr_grpo's max_completion_length; dapo's world size (N counts every rank)


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops as o
    return o


def _case(B, C, mu, beta, seed):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, C, generator=g) * 4
    old = lp + torch.randn(B, C, generator=g) * 0.2 if mu > 1 else None
    ref = lp + torch.randn(B, C, generator=g) * 0.3 if beta > 0 else None
    o = lp if old is None else old
    samp = o + torch.randn(B, C, generator=g) * 0.9
    adv = torch.randn(B, generator=g)
    mask = (torch.arange(C)[None, :] < torch.randint(1, C + 1, (B, 1), generator=g)).int()
    ent = torch.rand(B, C, generator=g) * 3
    if B > 2:
        mask[1] = 0                                                   # m = 0 row
        adv[2] = 0.0                                                  # A = 0 row: every token ties
    if old is not None and B > 3:
        old[3] = lp[3]                                                # ratio exactly 1: ties at the bound 1 + eps_high = 1
    return lp, old, ref, samp, adv, mask, ent


def _norm(loss_type, B, mask, n_items):
    if loss_type == "grpo":
        return dict(norm_rows=B), None
    d = dict(bnpo=max(float(mask.sum()), 1.0), dr_grpo=float(B * MAXLEN), dapo=max(n_items, 1.0) / WORLD)[loss_type]
    return dict(norm=torch.tensor([d], device="cuda")), d


def _near_kink(s64, m, lo, hi, delta, seq):
    """Tokens whose float64 ratio lies within 1e-5 (relative) of a clip bound or delta but not on it: fp32 rounding may take the other
    branch of min / clamp there, a jump of the gradient, not an error.  Ratios of exactly 1 (the designed ties) are kept."""
    c = torch.exp(s64)
    near = torch.zeros_like(c, dtype=torch.bool)
    for b in [1 - lo, 1 + hi] + ([delta] if delta is not None else []):
        near |= ((c - b).abs() <= 1e-5 * b) & (s64 != 0)
    return near & (m != 0) if not seq else near.expand_as(m) & (m != 0)


@pytest.mark.parametrize("level", ["token", "sequence"])
@pytest.mark.parametrize("loss_type", LOSS_TYPES)
def test_objective_kernel_vs_fp64(ops, loss_type, level):
    seq = level == "sequence"
    worst = 0.0
    for si, (B, C) in enumerate(SHAPES):
        for mu in (1, 2):
            for beta in (0.0, 0.04):
                lp, old, ref, samp, adv, mask, ent = _case(B, C, mu, beta, seed=100 * si + 10 * mu + int(beta > 0))
                lo, hi = (0.2, 0.0) if mu > 1 and B > 3 else (0.2, 0.28)
                n_items = float(mask.sum()) * 1.5                     # the other rank's tokens
                norm_kw, D = _norm(loss_type, B, mask, n_items)
                for delta in (None, 1.15):
                    for tis in (False, True):
                        for use_ent in (False, True):
                            cu = lambda t: None if t is None else t.cuda()
                            tau = torch.tensor([1.2]) if use_ent else None
                            out7, is_sums, ent_sum, dlp = ops.grpo_objective_raw(
                                lp.cuda(), cu(old), cu(ref), adv.cuda(), mask.cuda(), beta, lo, hi, sequence_level=seq, delta=delta,
                                rollout_lp=samp.cuda() if tis else None, is_cap=2.0, entropy=ent.cuda() if use_ent else None,
                                tau=cu(tau), **norm_kw)
                            keep = (ent >= tau) if use_ent else None
                            want = objective_with_grad(lp, old, ref, adv, mask, beta, lo, hi, loss_type=loss_type, level=level, delta=delta,
                                                       rollout=samp if tis else None, cap=2.0, keep=keep, max_completion_length=MAXLEN,
                                                       num_items=n_items, world=WORLD)
                            T = token_terms(lp.double(), None if old is None else old.double(), None if ref is None else ref.double(),
                                            adv.double(), mask, beta, lo, hi, level=level, delta=delta,
                                            rollout=samp.double() if tis else None, keep=keep)
                            m = mask.double()
                            # the loss against the scale of its summed terms (a sum near 0 is a cancellation, not a relative quantity)
                            absper = (T["per"].abs() * m).detach()
                            scale = (absper.sum(1) / T["nrm"]).sum() / B if loss_type == "grpo" else absper.sum() / D
                            o = lp.double() if old is None else old.double()
                            s64 = ((lp.double() - o) * m).sum(1, keepdim=True) / T["nrm"][:, None] if seq else lp.double() - o
                            near = _near_kink(s64, m, lo, hi, delta, seq)
                            tag = (B, C, mu, beta, delta, tis, use_ent)
                            got = out7.cpu().double()
                            assert abs(got[0] - want["loss"]) <= 2e-5 * scale + 1e-12, (tag, got[0].item(), want["loss"].item())
                            n = max(float(mask.sum()), 1.0)
                            if beta > 0:
                                assert abs(got[1] / B - want["kl"]) <= 2e-5 * want["kl"] + 1e-9, tag
                            slack = float(near.sum()) / n
                            for j, k in ((2, "clip"), (3, "low"), (4, "high"), (5, "region")):
                                assert abs(got[j] / n - want[k]) <= 1e-6 + slack, (tag, k)
                            assert got[6] == float(mask.sum())
                            ok = ~near
                            torch.testing.assert_close(dlp.cpu().double()[ok], want["dlp"][ok], rtol=2e-5, atol=1e-9)
                            assert torch.all(dlp.cpu()[mask == 0] == 0)
                            if tis:
                                st = is_sums.cpu().double() / n
                                for j in (0, 2, 3):
                                    assert abs(st[j] - want["is_stats"][j]) <= 2e-5 * max(1.0, abs(want["is_stats"][j].item())) + 1e-7, (tag, j)
                                assert abs(st[1] - want["is_stats"][1]) <= 1e-6 + 2.0 / n, tag
                            if use_ent:
                                assert abs(ent_sum.item() - float((ent.double() * m).sum())) <= 2e-5 * float((ent.double() * m).sum()) + 1e-6
                            worst = max(worst, float(abs(got[0] - want["loss"]) / (scale + 1e-30)))
    print(f"{loss_type}/{level}: worst loss err / scale {worst:.3g}")


@pytest.mark.parametrize("beta", [0.0, 0.04])
@pytest.mark.parametrize("mu", [1, 2])
def test_defaults_give_the_existing_kernels_bits(ops, mu, beta):
    for B, C in [(1, 7), (3, 512), (8, 512), (33, 4096), (40, 33)]:
        lp, old, ref, samp, adv, mask, ent = _case(B, C, mu, beta, seed=B + C + mu)
        cu = lambda t: None if t is None else t.cuda()
        args = (lp.cuda(), cu(old), cu(ref))
        n = torch.tensor(float(mask.sum()), device="cuda")
        Bt = torch.tensor(float(B), device="cuda")
        tau = torch.tensor([1.2], device="cuda")
        # plain
        a3, ad = ops.grpo_loss_raw(*args, adv.cuda(), mask.cuda(), beta, 0.2, 0.28)
        o7, _, _, od = ops.grpo_objective_raw(*args, adv.cuda(), mask.cuda(), beta, 0.2, 0.28, norm_rows=B)
        assert torch.equal(o7[0], a3[0]) and torch.equal(o7[1] / Bt, a3[1]) and torch.equal(o7[2] / n, a3[2]) and torch.equal(od, ad)
        # IS
        a3, ast, ad = ops.grpo_loss_is_raw(*args, samp.cuda(), adv.cuda(), mask.cuda(), beta, 0.2, 0.28, 2.0)
        o7, isum, _, od = ops.grpo_objective_raw(*args, adv.cuda(), mask.cuda(), beta, 0.2, 0.28, norm_rows=B, rollout_lp=samp.cuda(), is_cap=2.0)
        assert torch.equal(o7[0], a3[0]) and torch.equal(o7[2] / n, a3[2]) and torch.equal(od, ad) and torch.equal(isum / n, ast)
        # entropy, with and without IS
        for r in (None, samp.cuda()):
            a3, ast, aes, ad = ops.grpo_loss_ent_raw(*args, r, adv.cuda(), mask.cuda(), ent.cuda(), tau, beta, 0.2, 0.28, 2.0)
            o7, isum, oes, od = ops.grpo_objective_raw(*args, adv.cuda(), mask.cuda(), beta, 0.2, 0.28, norm_rows=B, rollout_lp=r,
                                                       is_cap=2.0, entropy=ent.cuda(), tau=tau)
            assert torch.equal(o7[0], a3[0]) and torch.equal(od, ad) and torch.equal(oes, aes)
            if r is not None:
                assert torch.equal(isum / n, ast)


def test_sequence_equals_token_level_at_mu1(ops):
    for B, C in [(3, 7), (8, 512), (33, 4096)]:
        lp, _, ref, _, adv, mask, _ = _case(B, C, 1, 0.04, seed=7 + B)
        for lt in LOSS_TYPES:
            kw, _ = _norm(lt, B, mask, float(mask.sum()))
            t7, _, _, td = ops.grpo_objective_raw(lp.cuda(), None, ref.cuda(), adv.cuda(), mask.cuda(), 0.04, 0.2, 0.28, **kw)
            s7, _, _, sd = ops.grpo_objective_raw(lp.cuda(), None, ref.cuda(), adv.cuda(), mask.cuda(), 0.04, 0.2, 0.28, sequence_level=True, **kw)
            torch.testing.assert_close(s7, t7, rtol=2e-5, atol=1e-7)
            torch.testing.assert_close(sd, td, rtol=2e-5, atol=1e-9)


def test_objective_refuses_bad_arguments(ops):
    lp, old, ref, samp, adv, mask, _ = _case(4, 8, 2, 0.04, seed=1)
    a = (lp.cuda(), old.cuda(), ref.cuda(), adv.cuda(), mask.cuda(), 0.04, 0.2, 0.2)
    for d in (0.0, -1.0, float("nan")):
        with pytest.raises(RuntimeError, match="delta"):
            ops.grpo_objective_raw(*a, norm_rows=4, delta=d)
    with pytest.raises(RuntimeError, match="is_cap"):
        ops.grpo_objective_raw(*a, norm_rows=4, rollout_lp=samp.cuda(), is_cap=0.0)


# ------------------------------------------------------------------ advantages and the truncated mask
@pytest.mark.parametrize("rows,G,nf", [(8, 4, 1), (64, 8, 3), (512, 16, 2), (96, 32, 1), (4096, 2, 2)])
def test_advantages_scaled(ops, rows, G, nf):
    g = torch.Generator().manual_seed(rows + G)
    r = torch.randn(rows, nf, generator=g) * 3
    r[:G] = 1.0                                                        # a zero-std group
    a_grp, gm, gs = ops.grpo_advantages(r.cuda(), G, return_stats=True)
    adv, sd, zero = ops.grpo_advantages_scaled(r.cuda(), G, "group")
    assert torch.equal(adv, a_grp) and torch.equal(sd, gs.repeat_interleave(G))
    assert zero[:G].all() and int(zero.sum()) == int((gs <= 1e-8).sum()) * G
    for mode in ("batch", "none"):
        adv, sd, zero = ops.grpo_advantages_scaled(r.cuda(), G, mode)
        wa, ws, wz = adv_ref(r, G, mode)
        torch.testing.assert_close(adv.cpu().double(), wa, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(sd.cpu().double(), ws, rtol=1e-5, atol=1e-6)
        assert torch.equal(zero.cpu().bool(), wz)


def test_eos_mask_truncated(ops):
    g = torch.Generator().manual_seed(3)
    for B, C in [(1, 1), (5, 7), (33, 300)]:
        ids = torch.randint(2, 40, (B, C), generator=g)
        ids[torch.arange(B), torch.randint(0, C, (B,), generator=g)] = 1             # every row holds an EOS
        m0 = ops.eos_mask(ids.cuda(), 1)
        m1, n1 = ops.eos_mask_truncated(ids.cuda(), 1)
        assert torch.equal(m0, m1) and torch.equal(n1, m0.sum(1).int())
        ids[::2] = torch.where(ids[::2] == 1, 2, ids[::2])                              # even rows truncated
        m1, n1 = ops.eos_mask_truncated(ids.cuda(), 1)
        wm, wn = truncated_mask(ids, 1)
        assert torch.equal(m1.cpu(), wm) and torch.equal(n1.cpu(), wn) and (m1[::2] == 0).all()


# ------------------------------------------------------------------ trainer
def _token_reward(completion_ids, **kw):
    return (completion_ids % 7 == 0).float().sum(1) - 0.1 * (completion_ids % 5 == 0).float().sum(1)


def _trainer(size="small", mu=1, maxlen=12, share=False, suppress=False, **fields):
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config(size), dna_config(size)
    oracle = build_oracle(tc, dc, seed=11)
    batch = (synth_batch(tc, dc, batch=4, n_seq=2, dna_len=50, text_len=60, seed=8, same_prompt=True) if size == "small" else
             synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14, same_prompt=True))
    m = DNALLMModel.from_oracle(oracle)
    cfg = DNALLMGRPOConfig(num_generations=4, max_completion_length=maxlen, per_device_train_batch_size=4, learning_rate=1e-2, lora_r=16,
                           lora_alpha=32.0, num_iterations=mu, beta=0.04, share_prompt_prefix=share, suppress_eos=suppress, **fields)
    tr = DNALLMGRPOTrainer(m, [_token_reward], cfg)
    with torch.no_grad():
        g = torch.Generator().manual_seed(5)
        for p in m._lora.params[1::2]:
            p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device))
    m.sync_adapters(rollout=True)
    return tr, m, batch, oracle


def _inputs(tr, m, batch, maxlen=12):
    inputs = tr._generate_and_score_completions(batch, m, uniforms=torch.rand(maxlen, 4, generator=torch.Generator().manual_seed(0)).cuda())
    inputs["advantages"] = torch.tensor([1.0, -0.5, 0.3, -0.8], device="cuda")
    return inputs


def _run(tr, m, inputs, **args):
    for k, v in args.items():
        setattr(tr.args, k, v)
    tr._step, tr.global_step = 0, 0
    tr._metrics.clear()
    m.zero_grad_buffers()
    loss = tr.compute_loss(m, inputs)
    return loss.clone(), [m._lora.flat_grad.clone(), m._proj_grad_w.clone(), m._proj_grad_b.clone()], \
        {k: [float(x) for x in v] for k, v in tr._metrics.items()}


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp(min=1e-30)).item()


@pytest.mark.parametrize("fields,mu", [(dict(loss_type="grpo"), 1), (dict(loss_type="bnpo"), 1), (dict(loss_type="dr_grpo"), 1),
                                       (dict(loss_type="dapo"), 1), (dict(importance_sampling_level="sequence"), 2),
                                       (dict(loss_type="dapo", importance_sampling_level="sequence", delta=1.05), 2)])
def test_training_step_vs_fp32_oracle(fields, mu):
    """The trainer's loss and LoRA / projector gradients against autograd of the contract on the fp32 oracle's log-probs (same
    adapters; old and reference log-probs are the trainer's, as data)."""
    from oracle import grpo as og, lora as olora
    tr, m, batch, oracle = _trainer(mu=mu, **fields)
    inputs = _inputs(tr, m, batch)
    # rows of different lengths, so that the four normalisers differ (the old / ref log-probs stay data; dapo recounts N)
    lens = torch.tensor([12, 7, 3, 10], device="cuda")
    inputs["completion_mask"] = inputs["completion_mask"] * (torch.arange(inputs["completion_mask"].shape[1], device="cuda")[None, :] < lens[:, None]).int()
    inputs.pop("num_items_in_batch", None)
    loss, _, met = _run(tr, m, inputs)
    m.attach_grads()
    comp, cmask = inputs["completion_ids"].cpu(), inputs["completion_mask"].cpu()
    C = comp.shape[1]
    olora.inject(oracle.text_model, 16, 32.0)
    sd = {k: v.detach().float().cpu() for k, v in m.text_model.state_dict().items() if "lora_" in k}
    assert not oracle.text_model.load_state_dict(sd, strict=False).unexpected_keys
    for p in oracle.dna_projection.parameters():
        p.requires_grad_(True)
    ids = torch.cat([batch["input_ids"], comp], 1)
    mask = torch.cat([batch["attention_mask"], cmask.long()], 1)
    mm = dict(dna_tokenized=batch["dna_tokenized"], batch_idx_map=batch["batch_idx_map"])
    lp_o = og.per_token_logps(oracle, ids, mask, **mm)[:, -C:]
    f = lambda t: None if t is None else t.detach().cpu().float()
    want = objective(lp_o, f(inputs["old_per_token_logps"]), f(inputs["ref_per_token_logps"]), inputs["advantages"].cpu(), cmask, 0.04,
                     0.2, 0.2, loss_type=tr.args.loss_type, level=tr.args.importance_sampling_level, delta=tr.args.delta,
                     max_completion_length=tr.max_completion_length, num_items=float(cmask.sum()), world=1)
    want["loss"].backward()
    assert abs(loss.item() - want["loss"].item()) < 5e-3, (loss.item(), want["loss"].item())
    onames = dict(oracle.text_model.named_parameters())
    worst = max(_rel(p.grad.cpu(), onames[n].grad) for n, p in m.text_model.named_parameters() if "lora_" in n)
    rw = _rel(m.dna_projection.weight.grad.cpu(), oracle.dna_projection.weight.grad)
    rb = _rel(m.dna_projection.bias.grad.cpu(), oracle.dna_projection.bias.grad)
    print(f"{fields} mu={mu}: loss {loss.item():.6f} vs {want['loss'].item():.6f}; LoRA grad rel {worst:.4f}; projector {rw:.4f} {rb:.4f}")
    assert worst < 0.08 and rw < 0.05 and rb < 0.05
    if tr.args.loss_type != "grpo" or mu > 1:
        assert {"clip_ratio/low_mean", "clip_ratio/high_mean", "clip_ratio/region_mean"} <= set(met)


def test_dapo_and_dr_grpo_equal_bnpo_bits():
    """World 1 without truncation: dapo's N / world is bnpo's token count.  Fixed-length rows (suppress_eos): dr_grpo's
    B * max_completion_length is that count too."""
    tr, m, batch, _ = _trainer(size="tiny", maxlen=8, suppress=True, loss_type="bnpo")
    inputs = _inputs(tr, m, batch, maxlen=8)
    assert inputs["completion_mask"].shape[1] == 8 and bool(inputs["completion_mask"].all())
    l_b, g_b, _ = _run(tr, m, inputs, loss_type="bnpo")
    for lt in ("dapo", "dr_grpo"):
        inp = dict(inputs)
        l, g, _ = _run(tr, m, inp, loss_type=lt)
        assert torch.equal(l, l_b) and all(torch.equal(a, b) for a, b in zip(g, g_b)), lt
    # and the dapo normaliser from the rollout is the count of the mask
    tr.args.loss_type = "dapo"
    inp = _inputs(tr, m, batch, maxlen=8)
    assert inp["num_items_in_batch"].item() == float(inp["completion_mask"].sum())


@pytest.mark.parametrize("share", [False, True])
def test_truncated_rows_get_no_gradient(share, monkeypatch):
    from bioreason_b200 import training
    tr, m, batch, _ = _trainer(size="tiny", maxlen=8, share=share, mask_truncated_completions=True, loss_type="bnpo")
    first = _inputs(tr, m, batch, maxlen=8)["completion_ids"].cpu()
    # an EOS token that row 0 emits and row 1 never does: row 0 ends there, row 1 (same draws) runs to the end
    tok = next(int(t) for t in first[0].tolist() if int(t) not in first[1].tolist())
    tr.eos_token_id = tok
    tr.generation_kwargs["eos_token_id"] = tok
    tr._metrics.clear()
    inputs = _inputs(tr, m, batch, maxlen=8)
    comp, cmask = inputs["completion_ids"].cpu(), inputs["completion_mask"].cpu()
    truncated = ~(comp == tok).any(1)
    assert truncated[1] and not truncated[0]
    assert (cmask[truncated] == 0).all() and (cmask[~truncated].sum(1) > 0).all()
    want_len = torch.where(truncated, torch.full((4,), comp.shape[1]), (comp == tok).int().argmax(1) + 1).float().mean()
    assert abs(float(tr._metrics["completion_length"][0]) - want_len.item()) < 1e-6
    seen = []
    orig = training.policy_backward
    monkeypatch.setattr(training, "policy_backward", lambda mdl, ctx, dlp, **k: (seen.append(dlp.clone()), orig(mdl, ctx, dlp, **k))[1])
    loss, grads, met = _run(tr, m, inputs)
    dlp = torch.cat(seen).cpu()
    assert (dlp[truncated] == 0).all() and (dlp[~truncated] != 0).any()
    assert torch.isfinite(loss) and all(torch.isfinite(g).all() and torch.any(g != 0) for g in grads)


@pytest.mark.parametrize("combo", ["tis", "entropy", "fp8", "dropout", "ga2", "share", "scale_batch", "scale_none"])
def test_objective_steps_compose(combo):
    kw = dict(tis=dict(rollout_is_correction=True), entropy=dict(top_entropy_quantile=0.3), fp8=dict(fp8_rollout=True),
              dropout=dict(apply_lora_dropout=True, lora_dropout=0.1, micro_rows=2), ga2=dict(gradient_accumulation_steps=2),
              share=dict(share=True, micro_rows=4), scale_batch=dict(scale_rewards="batch"), scale_none=dict(scale_rewards=False))[combo]
    tr, m, batch, _ = _trainer(size="tiny", maxlen=8, mu=2, loss_type="dapo", importance_sampling_level="sequence", delta=2.0,
                               mask_truncated_completions=True, **kw)
    for _ in range(2 * tr.args.gradient_accumulation_steps):
        assert torch.isfinite(tr.training_step(batch))
    met = tr.log_metrics()
    assert {"clip_ratio/low_mean", "clip_ratio/high_mean", "clip_ratio/region_mean", "clip_ratio", "kl"} <= set(met)
    # entropy/threshold is +inf when no token is valid (every tiny-model completion may be truncated)
    assert all(math.isfinite(v) for k, v in met.items() if k != "entropy/threshold")
    if combo.startswith("scale"):
        assert 0.0 <= met["frac_reward_zero_std"] <= 1.0
