"""Rollout log-probs and truncated importance sampling (TIS): the sampler's behaviour log-prob against float64 with a per-element
bound, the rollout plumbing (ids unchanged, graph == eager, EOS, FP8 == bf16 on grid-exact weights, accuracy against the fp32
oracle), the TIS loss kernel against the float64 restatement in rollout_is_ref.py, and the trainer flag."""
import math

import pytest
import torch

from rollout_is_ref import grpo_loss_is_with_grad

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24                      # fp32 unit roundoff
CHUNK = 4096                          # logits per stage-1 CTA of the two-stage sampler


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops as o
    return o


# ------------------------------------------------------------------ 1. sampler log-prob vs float64
MODES = {                              # name -> (do_sample, top_k, two-stage workspace)
    "greedy": (False, 20, True),
    "sampled": (True, 20, True),
    "topk64": (True, 64, True),        # top_k > 32: the single-stage sampler, workspace or not
    "greedy_1stage": (False, 20, False),
}
# randn1 lifts the tail chunk by 2 so that a reference that drops it is visibly wrong even when the tail is one logit
FAMILIES = ["randn1", "randn10", "randn30", "spike80", "ties", "neginf_chunks", "finished"]


def make_logits(fam, R, V, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(R, V, device="cuda", generator=g)
    if fam.startswith("randn"):
        z *= float(fam[5:])
        if fam == "randn1" and V > CHUNK:
            z[:, (V // CHUNK) * CHUNK:] += 2.0
    elif fam == "spike80":
        z[torch.arange(R), torch.randint(0, V, (R,), device="cuda", generator=g)] = 80.0
    elif fam == "ties":
        z = torch.randint(0, 3, (R, V), device="cuda", generator=g).float()
    elif fam == "neginf_chunks":
        z *= 3
        n_chunks = (V + CHUNK - 1) // CHUNK
        if n_chunks > 1:
            for c in range(0, n_chunks - 1, 2):                               # whole chunks, the tail chunk stays finite
                z[:, c * CHUNK:(c + 1) * CHUNK] = -math.inf
        else:
            z[:, : V // 2] = -math.inf
    finished = torch.zeros(R, device="cuda", dtype=torch.int32)
    if fam == "finished":
        finished[1::2] = 1
    return z, finished


def run_sampler(ops, z, finished, mode, seed, logp=True):
    do_sample, top_k, two_stage = MODES[mode]
    R, V = z.shape
    u = torch.rand(1, R, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
    tok = torch.full((R, 1), -7, device="cuda", dtype=torch.int64)
    lp = torch.full((R, 1), float("nan"), device="cuda") if logp else None
    fin = finished.clone()
    ws = ops.sample_workspace(R, V, "cuda", logp=True) if two_stage else None
    ops.sample_next(z, workspace=ws, temperature=0.6, top_k=top_k, top_p=0.95, do_sample=do_sample, uniforms=u if do_sample else None,
                    max_steps=1, eos_id=-1, pad_id=0, finished=fin, tokens=tok, logp=lp)
    return tok[:, 0], (lp[:, 0] if logp else None)


def logp_bound(z64, y, logp_ref):
    """Per-element bound on |fp32 logp - float64 logp|: the exp arguments (u |z - M| per term, twice: chunk and combine), the exps
    and products (12 u), the summation depth, log S, M + log S and the final subtraction, times a safety factor of 2."""
    R, V = z64.shape
    M = z64.max(1).values
    t = torch.exp(z64 - M[:, None])
    S = t.sum(1)
    A = torch.where(t > 0, t * (z64 - M[:, None]).abs(), torch.zeros_like(t)).sum(1)
    depth = math.ceil(V / 1024) + 16 + 10 + math.ceil(V / CHUNK / 32) + 5
    lse = M + torch.log(S)
    return 2 * U32 * (depth + 12 + 2 * A / S + 2 * torch.log(S).abs() + lse.abs() + logp_ref.abs())


@pytest.mark.parametrize("V", [151936, 3 * 4096 + 1, 1000])
@pytest.mark.parametrize("R", [1, 3, 8, 32])
def test_sampler_logp_vs_fp64(ops, R, V):
    worst = 0.0
    for mode in MODES:
        for fi, fam in enumerate(FAMILIES):
            seed = 1000 * R + 10 * fi + len(mode)
            z, finished = make_logits(fam, R, V, seed)
            tok0, _ = run_sampler(ops, z, finished, mode, seed, logp=False)
            tok, lp = run_sampler(ops, z, finished, mode, seed)
            tok2, lp2 = run_sampler(ops, z, finished, mode, seed)
            # the output does not change the draw (past 1024 ties of the k-th value the kept ties are the lowest ids: deterministic)
            assert torch.equal(tok, tok0) and torch.equal(tok, tok2), (mode, fam)
            assert torch.equal(lp.view(torch.int32), lp2.view(torch.int32)), (mode, fam)
            done = finished.bool()
            assert torch.all(lp[done] == 0) and torch.all(tok[done] == 0), (mode, fam)
            live = ~done
            if mode.startswith("greedy"):
                zm = z.masked_fill(torch.isinf(z), -3e38)
                assert torch.equal(z[live].gather(1, tok[live, None])[:, 0], zm[live].max(1).values), (mode, fam)
            z64 = z.double()[live]
            y = tok[live]
            ref = z64.gather(1, y[:, None])[:, 0] - torch.logsumexp(z64, 1)
            bound = logp_bound(z64, y, ref)
            err = (lp[live].double() - ref).abs()
            assert torch.all(torch.isfinite(lp[live])), (mode, fam)
            assert torch.all(err <= bound), (mode, fam, (err / bound).max().item())
            worst = max(worst, (err / bound).max().item())
            if fam == "randn1":
                # references that get the definition wrong exceed the bound
                zy = z64.gather(1, y[:, None])[:, 0]
                wrong = {"T=0.6": zy - torch.logsumexp(z64 / 0.6, 1),
                         "top-k only": zy - torch.logsumexp(z64.topk(min(20, V), 1).values, 1)}
                if V > CHUNK:
                    wrong["no tail chunk"] = zy - torch.logsumexp(z64[:, : (V // CHUNK) * CHUNK], 1)
                for name, w in wrong.items():
                    assert torch.any((lp[live].double() - w).abs() > bound), (mode, name)
    print(f"R={R} V={V}: worst err/bound {worst:.3f}")


def test_sampler_logp_refuses_a_small_workspace(ops):
    z = torch.randn(2, 151936, device="cuda")
    tok = torch.zeros(2, 1, device="cuda", dtype=torch.int64)
    lp = torch.zeros(2, 1, device="cuda")
    with pytest.raises(AssertionError, match="logp=True"):
        ops.sample_next(z, workspace=ops.sample_workspace(2, 151936, "cuda"), do_sample=False, tokens=tok, logp=lp)


# ------------------------------------------------------------------ 2. rollout
def _gen(m, batch, logp, **kw):
    out = m.generate(**batch, return_logprobs=logp, **kw)
    return (out[0].cpu(), out[1].cpu()) if logp else (out.cpu(), None)


def test_rollout_logprobs_plumbing():
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config("small"), dna_config("small")
    m = DNALLMModel.from_oracle(build_oracle(tc, dc, seed=5))
    g4 = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=50, text_len=60, seed=8, same_prompt=True)       # G = 4, shared pages
    g1 = synth_batch(tc, dc, batch=3, n_seq=1, dna_len=[9, 7, 9], text_len=[40, 25, 33], seed=9)       # G = 1, two lengths
    two = [synth_batch(tc, dc, batch=2, n_seq=1, dna_len=9, text_len=n, seed=s, same_prompt=True) for n, s in ((40, 21), (70, 22))]
    C = 10
    for batch in [g4, g1] + two:
        B = batch["input_ids"].shape[0]
        u = torch.rand(C, B, generator=torch.Generator().manual_seed(B))
        for kw in (dict(do_sample=False), dict(do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u)):
            res = {}
            for use_graph in (False, True):
                ids0, _ = _gen(m, batch, False, max_new_tokens=C, use_graph=use_graph, **kw)
                ids, lp = _gen(m, batch, True, max_new_tokens=C, use_graph=use_graph, **kw)
                assert torch.equal(ids, ids0) and lp.shape == ids.shape and lp.dtype == torch.float32
                assert torch.all(torch.isfinite(lp)) and torch.all(lp <= 0)
                res[use_graph] = lp
            assert torch.equal(res[False].view(torch.int32), res[True].view(torch.int32))      # graph and eager bit-identical
        # EOS: the token greedy decoding emits at step 3 ends that row there; everything after it is 0.0
        ids, _ = _gen(m, batch, False, max_new_tokens=8, do_sample=False)
        eos = int(ids[0, 3])
        for use_graph in (False, True):
            kw = dict(max_new_tokens=8, do_sample=False, eos_token_id=eos, pad_token_id=0, use_graph=use_graph)
            ids0, _ = _gen(m, batch, False, **kw)
            ids, lp = _gen(m, batch, True, **kw)
            assert torch.equal(ids, ids0)
            for r in range(ids.shape[0]):
                hit = (ids[r] == eos).nonzero()
                if len(hit):
                    e = int(hit[0])
                    assert torch.isfinite(lp[r, e]) and lp[r, e] <= 0
                    assert torch.all(lp[r, e + 1:] == 0)
    # the stats tuple comes last
    ids, lp, st = m.generate(**g4, max_new_tokens=4, do_sample=False, return_logprobs=True, return_stats=True)
    assert st["G"] == 4 and lp.shape == ids.shape


def test_rollout_logprobs_accuracy_vs_fp32_oracle():
    """LoRA B != 0: the rollout samples through merged, folded decode weights; its log-probs are compared with the fp32 oracle's
    log-probs of the same completions, and with the error of the trainer's own scoring pass (per_token_logps)."""
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from oracle import grpo as og, lora as olora
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config("small"), dna_config("small")
    oracle = build_oracle(tc, dc, seed=11)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=50, text_len=60, seed=8, same_prompt=True)
    m = DNALLMModel.from_oracle(oracle)
    lora = m.enable_lora(r=16, alpha=32.0, seed=3)
    with torch.no_grad():
        g = torch.Generator().manual_seed(5)
        for p in lora.params[1::2]:
            p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device))
    m.sync_adapters(rollout=True)
    olora.inject(oracle.text_model, 16, 32.0)
    sd = {k: v.detach().float().cpu() for k, v in m.text_model.state_dict().items() if "lora_" in k}
    _, unexpected = oracle.text_model.load_state_dict(sd, strict=False)
    assert not unexpected
    C = 16
    u = torch.rand(C, 4, generator=torch.Generator().manual_seed(2))
    ids, lp_roll = m.generate(**batch, max_new_tokens=C, do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u,
                              return_logprobs=True)
    ids, lp_roll = ids.cpu(), lp_roll.cpu()
    Cc = ids.shape[1]
    cmask = og.completion_mask_from_eos(ids, tc.eos_token_id)
    full_ids = torch.cat([batch["input_ids"], ids], 1)
    full_mask = torch.cat([batch["attention_mask"], cmask.long()], 1)
    mm = dict(dna_tokenized=batch["dna_tokenized"], batch_idx_map=batch["batch_idx_map"])
    with torch.no_grad():
        lp_o = og.per_token_logps(oracle, full_ids, full_mask, **mm)[:, -Cc:]
        lp_own = m.per_token_logps(full_ids, full_mask, batch["dna_tokenized"], batch["batch_idx_map"], keep_last=Cc).cpu()
    att = cmask.bool()
    e_roll = (lp_roll - lp_o)[att].abs().max().item()
    e_own = (lp_own - lp_o)[att].abs().max().item()
    print(f"rollout log-prob max err vs fp32 oracle {e_roll:.4e}, scoring pass {e_own:.4e}, ratio {e_roll / e_own:.3f}")
    assert e_roll <= 2 * e_own


# grid-exact weights (copied from test_gpu_fp8_rollout.py): the FP8 decode computes the same products as the bf16 one
E4M3 = torch.float8_e4m3fn


def grid_matrix(N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = 2.0 ** torch.randint(-14, -8, (N, 1), device="cuda", generator=g).float()
    q = (torch.randn(N, K, device="cuda", generator=g) * 60).clamp(-448, 448).to(E4M3).float()
    q[torch.arange(N), torch.randint(0, K, (N,), device="cuda", generator=g)] = 448.0
    return (q * s).bfloat16()


def grid_exact_oracle(size, seed):
    from bioreason_b200.configs import dna_config, text_config
    from oracle.models import build_oracle
    tc, dc = text_config(size), dna_config(size)
    oracle = build_oracle(tc, dc, seed=seed)
    sd = oracle.state_dict()
    with torch.no_grad():
        for i, (k, v) in enumerate(sorted(sd.items())):
            if not k.startswith("text_model.model.layers."):
                continue
            if k.endswith(("input_layernorm.weight", "post_attention_layernorm.weight")):
                v.fill_(1.0)
            elif k.endswith(("proj.weight",)) and ("self_attn" in k or "mlp" in k):
                v.copy_(grid_matrix(v.shape[0], v.shape[1], seed=seed * 1000 + i).to(v.device, v.dtype))
    return oracle, tc, dc


def test_fp8_rollout_logprobs_equal_bf16_on_grid_weights():
    from bioreason_b200.models import DNALLMModel
    from oracle.models import synth_batch
    oracle, tc, dc = grid_exact_oracle("small", seed=11)
    bf = DNALLMModel.from_oracle(oracle)
    f8 = DNALLMModel.from_oracle(oracle)
    f8.set_fp8_rollout(True)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=50, text_len=60, seed=8, same_prompt=True)
    C = 12
    u = torch.rand(C, 4, generator=torch.Generator().manual_seed(1))
    for kw in (dict(do_sample=False), dict(do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u)):
        for use_graph in (False, True):
            a_ids, a_lp = _gen(bf, batch, True, max_new_tokens=C, use_graph=use_graph, **kw)
            b_ids, b_lp = _gen(f8, batch, True, max_new_tokens=C, use_graph=use_graph, **kw)
            assert torch.equal(a_ids, b_ids) and torch.equal(a_lp.view(torch.int32), b_lp.view(torch.int32))


# ------------------------------------------------------------------ 3. loss kernel vs float64
def _loss_case(B, C, mu, beta, seed, empty_rows=True):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(B, C, generator=g) * 4
    old = lp + torch.randn(B, C, generator=g) * 0.2 if mu > 1 else None
    ref = lp + torch.randn(B, C, generator=g) * 0.3 if beta > 0 else None
    o = lp if old is None else old
    samp = o + torch.randn(B, C, generator=g) * 0.9                         # exp(o - b) on both sides of every cap
    adv = torch.randn(B, generator=g)
    mask = (torch.arange(C)[None, :] < torch.randint(1, C + 1, (B, 1), generator=g)).int()
    if empty_rows and B > 2:
        mask[1] = 0
    return lp, old, ref, samp, adv, mask


def _wrong_loss(kind, lp, old, ref, samp, adv, mask, beta, lo, hi, cap):
    """The TIS loss with one mistake, float64: the weight also on the KL term ("w_on_kl"), the weight differentiated through lp
    ("w_differentiated", mu = 1), or the cap applied to the log-ratio ("cap_on_log_ratio": exp(min(o - b, cap)))."""
    x = lp.double().clone().requires_grad_(True)
    o = x.detach() if old is None else old.double()
    m = mask.double()
    if kind == "w_differentiated":
        w = torch.clamp(torch.exp(x - samp.double()), max=cap)
    elif kind == "cap_on_log_ratio":
        w = torch.exp(torch.clamp(o - samp.double(), max=cap))
    else:
        w = torch.clamp(torch.exp(o - samp.double()), max=cap)
    c1 = torch.exp(x - o)
    c2 = torch.clamp(c1, 1 - lo, 1 + hi)
    a = adv.double()[:, None]
    per = -torch.min(c1 * a, c2 * a) * w
    if beta > 0:
        dk = ref.double() - x
        per = per + beta * (torch.exp(dk) - dk - 1) * (w if kind == "w_on_kl" else 1.0)
    cnt = m.sum(1)
    loss = torch.where(cnt > 0, (per * m).sum(1) / torch.where(cnt > 0, cnt, torch.ones_like(cnt)), torch.zeros_like(cnt)).mean()
    loss.backward()
    return loss.detach(), x.grad


CAPS = [0.5, 1.0, 2.0, math.inf]


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("beta,mu,lo,hi", [(0.04, 1, 0.2, 0.2), (0.04, 2, 0.2, 0.28), (0.0, 2, 0.1, 0.3), (0.0, 1, 0.2, 0.28)])
def test_is_loss_kernel_vs_fp64(ops, cap, beta, mu, lo, hi):
    for B, C in [(8, 512), (3, 7), (40, 33)]:
        lp, old, ref, samp, adv, mask = _loss_case(B, C, mu, beta, seed=B * 7 + C + mu)
        cu = lambda t: None if t is None else t.cuda()
        out3, stats, dlp = ops.grpo_loss_is_raw(lp.cuda(), cu(old), cu(ref), samp.cuda(), adv.cuda(), mask.cuda(), beta, lo, hi, cap)
        out3b, stats_b, dlp_b = ops.grpo_loss_is_raw(lp.cuda(), cu(old), cu(ref), samp.cuda(), adv.cuda(), mask.cuda(), beta, lo, hi, cap)
        assert torch.equal(out3, out3b) and torch.equal(stats, stats_b) and torch.equal(dlp, dlp_b)           # deterministic
        out3, stats, dlp = out3.cpu().double(), stats.cpu().double(), dlp.cpu().double()
        loss, kl, clip, st, grad = grpo_loss_is_with_grad(lp, old, ref, samp, adv, mask, beta, lo, hi, cap)
        # scalars: rtol 2e-5 of the scale of the summed terms (a mean near 0 is a cancellation, not a relative quantity)
        m = mask.double()
        o = (lp if old is None else old).double()
        d = o - samp.double()
        r = torch.exp(d)
        scales = [(torch.clamp(r, max=cap) * m).sum() / m.sum(), torch.ones(()), (d.abs() * m).sum() / m.sum(), ((r - 1 - d).abs() * m).sum() / m.sum()]
        for j in range(4):
            assert abs(stats[j] - st[j]) <= 2e-5 * scales[j] + 1e-7, (B, C, j, stats[j].item(), st[j].item())
        assert abs(out3[0] - loss) <= 2e-5 * max(1.0, abs(loss.item())), (B, C, out3[0].item(), loss.item())
        if beta > 0:
            assert abs(out3[1] - kl) <= 2e-5 * max(1e-3, abs(kl.item()))
        assert abs(out3[2] - clip) <= 1e-6
        torch.testing.assert_close(dlp, grad, rtol=2e-5, atol=1e-8)
        assert torch.all(dlp[mask == 0] == 0)
        if B * C > 100 and cap < math.inf:
            assert 0 < st[1] < 1                                             # weights on both sides of the cap
        # the wrong definitions fail the same check (on the shapes with enough tokens on both sides of the cap)
        for kind in ("w_on_kl", "w_differentiated", "cap_on_log_ratio") if B * C > 100 else ():
            if kind == "w_on_kl" and beta == 0:
                continue
            if kind == "w_differentiated" and old is not None:
                continue                                                     # with mu > 1 the weight has no lp dependence to differentiate
            if kind == "cap_on_log_ratio" and cap == math.inf:
                continue
            wl, wg = _wrong_loss(kind, lp, old, ref, samp, adv, mask, beta, lo, hi, cap)
            ok_loss = abs(out3[0] - wl) <= 2e-5 * max(1.0, abs(wl.item()))
            ok_grad = torch.allclose(dlp, wg, rtol=2e-5, atol=1e-8)
            assert not (ok_loss and ok_grad), (kind, B, C)


@pytest.mark.parametrize("beta", [0.0, 0.04])
def test_is_loss_with_unit_weights_equals_plain_loss(ops, beta):
    """mu = 2, rollout log-probs = old and cap = inf: every weight is exactly 1, so out3 and dlp are grpo_loss_raw's, bit for bit."""
    for B, C in [(8, 512), (3, 7), (40, 33)]:
        lp, old, ref, _, adv, mask = _loss_case(B, C, 2, beta, seed=B + C)
        cu = lambda t: None if t is None else t.cuda()
        a3, ad = ops.grpo_loss_raw(lp.cuda(), old.cuda(), cu(ref), adv.cuda(), mask.cuda(), beta, 0.2, 0.28)
        b3, st, bd = ops.grpo_loss_is_raw(lp.cuda(), old.cuda(), cu(ref), old.cuda(), adv.cuda(), mask.cuda(), beta, 0.2, 0.28, math.inf)
        assert torch.equal(a3, b3) and torch.equal(ad, bd)
        assert st.tolist() == [1.0, 0.0, 0.0, 0.0]


def test_is_loss_refuses_bad_arguments(ops):
    lp, old, ref, samp, adv, mask = _loss_case(4, 8, 2, 0.04, seed=1)
    args = [lp.cuda(), old.cuda(), ref.cuda(), samp.cuda(), adv.cuda(), mask.cuda(), 0.04, 0.2, 0.2]
    for cap in (0.0, -1.0, float("nan")):
        with pytest.raises(RuntimeError, match="is_cap"):
            ops.grpo_loss_is_raw(*args, cap)


# ------------------------------------------------------------------ 4. trainer
def _token_reward(completion_ids, **kw):
    return (completion_ids % 7 == 0).float().sum(1) - 0.1 * (completion_ids % 5 == 0).float().sum(1)


def _trainer(mu, share, beta, fp8=False, tis=False, cap=2.0, seed=21):
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config("tiny"), dna_config("tiny")
    oracle = build_oracle(tc, dc, seed=seed)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14, same_prompt=True)
    m = DNALLMModel.from_oracle(oracle)
    cfg = DNALLMGRPOConfig(num_generations=4, max_completion_length=6, per_device_train_batch_size=4, learning_rate=1e-2, lora_r=16,
                           lora_alpha=32.0, num_iterations=mu, beta=beta, share_prompt_prefix=share, micro_rows=4, fp8_rollout=fp8,
                           rollout_is_correction=tis, rollout_is_cap=cap)
    tr = DNALLMGRPOTrainer(m, [_token_reward], cfg)
    with torch.no_grad():                                                   # B != 0: the rollout and the trainer see live adapters
        g = torch.Generator().manual_seed(5)
        for p in m._lora.params[1::2]:
            p.copy_((torch.randn(p.shape, generator=g) * 0.02).to(p.device))
    m.sync_adapters(rollout=True)
    return tr, m, batch


def _grads(m):
    return [m._lora.flat_grad.clone(), m._proj_grad_w.clone(), m._proj_grad_b.clone()]


def _loss_and_grads(tr, m, inputs, tis):
    tr.args.rollout_is_correction = tis
    tr._step, tr.global_step = 0, 0
    tr._metrics.clear()
    m.zero_grad_buffers()
    loss = tr.compute_loss(m, inputs)
    return loss.clone(), _grads(m), {k: [float(x) for x in v] for k, v in tr._metrics.items()}


@pytest.mark.parametrize("share", [False, True])
def test_trainer_capped_weights_double_the_gradient(share):
    """beta = 0, mu = 1, one chunk, cap 2, rollout log-probs = the policy's own minus 1: every w is min(e, 2) = 2 exactly, so the loss
    and every gradient are exactly twice the uncorrected ones."""
    tr, m, batch = _trainer(1, share, 0.0)
    inputs = tr._generate_and_score_completions(batch, m, uniforms=torch.rand(6, 4, generator=torch.Generator().manual_seed(0)).cuda())
    assert "sampling_per_token_logps" not in inputs and "return_logprobs" not in tr.generation_kwargs
    ids = torch.cat([inputs["prompt_ids"], inputs["completion_ids"]], 1)
    mask = torch.cat([inputs["prompt_mask"], inputs["completion_mask"].to(inputs["prompt_mask"].dtype)], 1)
    C = inputs["completion_ids"].shape[1]
    own = tr._get_per_token_logps(m, ids, mask, keep_last=C, group_size=inputs["local_group_size"], **inputs["multimodal_inputs"])
    inputs["sampling_per_token_logps"] = own - 1.0
    inputs["advantages"] = torch.tensor([1.0, -0.5, 0.3, -0.8], device="cuda")  # non-zero whatever the rewards were
    l0, g0, _ = _loss_and_grads(tr, m, inputs, False)
    l1, g1, met = _loss_and_grads(tr, m, inputs, True)
    assert torch.equal(l1, 2 * l0)
    for a, b in zip(g0, g1):
        assert torch.any(a != 0) and torch.equal(b, 2 * a)
    assert met["rollout_is/capped_frac"] == [1.0] and met["rollout_is/ratio_mean"] == [2.0]
    assert abs(met["rollout_is/logp_diff"][0] - 1.0) < 1e-5


@pytest.mark.parametrize("share", [False, True])
def test_trainer_unit_weights_leave_the_gradient_unchanged(share):
    """mu = 2, rollout log-probs = old, cap = inf: w = 1 everywhere and the gradients are bit-identical to the uncorrected run."""
    tr, m, batch = _trainer(2, share, 0.04, cap=math.inf)
    inputs = tr._generate_and_score_completions(batch, m, uniforms=torch.rand(6, 4, generator=torch.Generator().manual_seed(0)).cuda())
    inputs["sampling_per_token_logps"] = inputs["old_per_token_logps"].clone()
    inputs["advantages"] = torch.tensor([1.0, -0.5, 0.3, -0.8], device="cuda")
    l0, g0, _ = _loss_and_grads(tr, m, inputs, False)
    l1, g1, met = _loss_and_grads(tr, m, inputs, True)
    assert torch.equal(l0, l1)
    for a, b in zip(g0, g1):
        assert torch.any(a != 0) and torch.equal(a, b)
    assert met["rollout_is/ratio_mean"] == [1.0] and met["rollout_is/capped_frac"] == [0.0] and met["rollout_is/kl"] == [0.0]


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("mu", [1, 2])
def test_training_steps_with_correction(fp8, mu):
    tr, m, batch = _trainer(mu, False, 0.04, fp8=fp8, tis=True, cap=2.0)
    assert tr.generation_kwargs["return_logprobs"] is True
    inputs = tr._generate_and_score_completions(batch, m)
    lp = inputs["sampling_per_token_logps"]
    assert lp.shape == inputs["completion_ids"].shape and torch.all(torch.isfinite(lp)) and torch.all(lp <= 0)
    for _ in range(2):
        assert torch.isfinite(tr.training_step(batch))
    met = tr.log_metrics()
    assert 0 < met["rollout_is/ratio_mean"] <= 2.0 and 0 <= met["rollout_is/capped_frac"] <= 1
    assert math.isfinite(met["rollout_is/logp_diff"]) and met["rollout_is/kl"] > -1e-6
    print(f"fp8={fp8} mu={mu}:", {k: round(v, 5) for k, v in met.items() if k.startswith("rollout_is/")})
