"""Parity at the shapes bench.py measures (VERDICT r1 'parity at the shapes you benchmark'): real Qwen3 / NT-v2 WIDTHS (d, F, heads,
V = 151 936), reduced DEPTH (2 decoder + 2 encoder layers keep the fp32 oracle affordable), the real sequence geometry of BASELINE
configs (b), (c), (e): L = 2360 with a G = 8 shared prefix, SFT batch 8, ragged left-padded KEGG-shape batches, an EOS-terminated rollout.

The oracle (HF classes, fp32, TEST INFRASTRUCTURE) runs on the same GPU in fp32 here -- it is the checker, not the product.
Budget regime (DESIGN.md §3): bf16 storage / fp32 accumulate cannot meet `logits rtol 1e-3` against an fp32 oracle; the bar is
"no further from the fp32 result than 1.25x the reference's OWN bf16 path on the same inputs"; integer work is bit-exact."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return (a.float() - b.float()).norm().item() / (b.float().norm().item() + 1e-12)


def _first_mismatch_ok(got, want, margins, tol):
    """Greedy ids must be bit-exact except where the oracle's own top-2 margin is below the bf16 noise floor; after such a near-tie
    flip the continuations legitimately diverge, so comparison of that row stops there."""
    n_flip = 0
    for r in range(want.shape[0]):
        for t in range(min(got.shape[1], want.shape[1])):
            if got[r, t] != want[r, t]:
                assert margins[r, t] < tol, f"row {r} step {t}: ids differ with oracle margin {margins[r, t]:.4f}"
                n_flip += 1
                break
    return n_flip


def _cfgs(text, depth=2):
    from bioreason_b200.configs import text_config, dna_config
    tc, dc = text_config(text), dna_config("nt-v2-500m")
    tc.num_hidden_layers = depth
    if hasattr(tc, "layer_types"):
        tc.layer_types = tc.layer_types[:depth]
    dc.num_hidden_layers = depth
    return tc, dc


def _cuda_batch(b):
    out = dict(input_ids=b["input_ids"].cuda(), attention_mask=b["attention_mask"].cuda(), batch_idx_map=b["batch_idx_map"])
    out["dna_tokenized"] = {k: v.cuda() for k, v in b["dna_tokenized"].items()} if b.get("dna_tokenized") else None
    return out


def _oracle_logps(oracle, ids, mask, mm, keep, rows_per_call=1):
    """per_token_logps row by row (the [B, L, V] fp32 logits of 8 x 2360 x 151936 would be 11 GB per copy)."""
    from oracle import grpo as og
    out = []
    B = ids.shape[0]
    for lo in range(0, B, rows_per_call):
        hi = min(B, lo + rows_per_call)
        idx = [i for i, b in enumerate(mm["batch_idx_map"]) if lo <= b < hi]
        dna = {k: v[idx] for k, v in mm["dna_tokenized"].items()}
        out.append(og.per_token_logps(oracle, ids[lo:hi], mask[lo:hi], dna_tokenized=dna, batch_idx_map=[mm["batch_idx_map"][i] - lo for i in idx])[:, -keep:])
    return torch.cat(out)


def _build_pair(tc, dc, seed, r=32, alpha=64.0, lora_seed=3):
    """(oracle fp32 on cuda with peft-shaped adapters, DNALLMModel with the same weights and adapters)"""
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle
    from oracle import lora as olora
    oracle = build_oracle(tc, dc, seed=seed)
    m = DNALLMModel.from_oracle(oracle)
    lora = m.enable_lora(r=r, alpha=alpha, seed=lora_seed)
    with torch.no_grad():                                                  # non-zero B so every gradient path is live
        g = torch.Generator().manual_seed(5)
        for p in lora.params[1::2]:
            p.copy_((torch.randn(p.shape, generator=g) * 0.01).to(p.device))
    m.sync_adapters(rollout=True)
    olora.inject(oracle.text_model, r, alpha)
    sd = {k: v.detach().float().cpu() for k, v in m.text_model.state_dict().items() if "lora_" in k}
    assert not oracle.text_model.load_state_dict(sd, strict=False).unexpected_keys
    oracle = oracle.cuda()
    for p in oracle.dna_projection.parameters():
        p.requires_grad_(True)
    return oracle, m, lora


def _grad_report(m, oracle):
    m.attach_grads()
    onames = dict(oracle.text_model.named_parameters())
    worst, worst_name = 0.0, ""
    for name, p in m.text_model.named_parameters():
        if "lora_" in name:
            rel = _rel(p.grad, onames[name].grad)
            if rel > worst:
                worst, worst_name = rel, name
    rw = _rel(m.dna_projection.weight.grad, oracle.dna_projection.weight.grad)
    rb = _rel(m.dna_projection.bias.grad, oracle.dna_projection.bias.grad)
    return worst, worst_name, rw, rb


def test_config_c_logps_grads_microrows_determinism():
    """Config (c) geometry: 1 prompt x G = 8, P = 1852 (2 x 668 DNA tokens + 4 delimiters + 512 text), C = 512, L = 2364, Qwen3-4B widths."""
    from bioreason_b200 import training
    from oracle.models import synth_batch
    tc, dc = _cfgs("qwen3-4b")
    oracle, m, lora = _build_pair(tc, dc, seed=31)
    G, C = 8, 512
    batch = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
    P = batch["input_ids"].shape[1]
    assert P == 512 + 2 * (668 + 2)                                        # text + per DNA sequence: <|dna_start|> 668 x <|dna_pad|> <|dna_end|>
    comp = torch.randint(0, tc.eos_token_id, (G, C), generator=torch.Generator().manual_seed(9))
    ids = torch.cat([batch["input_ids"], comp], 1).cuda()
    cmask = torch.ones(G, C, dtype=torch.long); cmask[1, -37:] = 0; cmask[5, -200:] = 0          # post-EOS tails
    mask = torch.cat([batch["attention_mask"], cmask], 1).cuda()
    wgt = (torch.randn(G, C, generator=torch.Generator().manual_seed(10)) * cmask).cuda()
    cb = _cuda_batch(batch)
    mm = dict(dna_tokenized=cb["dna_tokenized"], batch_idx_map=cb["batch_idx_map"])
    # ---- oracle fp32: log-probs + gradients, row by row
    lp_o = []
    for r in range(G):
        lp_r = _oracle_logps(oracle, ids[r:r + 1], mask[r:r + 1], dict(dna_tokenized={k: v[2 * r:2 * r + 2] for k, v in mm["dna_tokenized"].items()},
                                                                       batch_idx_map=[0, 0]), C)
        (lp_r * wgt[r:r + 1]).sum().backward()
        lp_o.append(lp_r.detach())
    lp_o = torch.cat(lp_o)
    # ---- the reference's own bf16 path (same module tree cast to bf16) sets the error budget
    o16 = copy.deepcopy(oracle).to(torch.bfloat16)
    with torch.no_grad():
        lp16 = torch.cat([_oracle_logps(o16, ids[r:r + 1], mask[r:r + 1], dict(dna_tokenized={k: v[2 * r:2 * r + 2] for k, v in mm["dna_tokenized"].items()},
                                                                                 batch_idx_map=[0, 0]), C).float() for r in range(G)])
    del o16
    # ---- CUDA path, in row chunks: the activations one row keeps for the backward at L = 2364 are ~9 GB (Qwen3-4B, 36 layers), so the
    #      8 rows do not fit next to the fp32 oracle on an 80 GB device.  Rows are independent in the forward and the loss is row-separable.
    def chunked(rows_per_chunk):
        lps = []
        for lo in range(0, G, rows_per_chunk):
            hi = lo + rows_per_chunk
            idx = [i for i, b in enumerate(mm["batch_idx_map"]) if lo <= b < hi]
            dna = {k: v[idx] for k, v in mm["dna_tokenized"].items()}
            lp_c, ctx = training.policy_forward(m, ids[lo:hi], mask[lo:hi], dna, [mm["batch_idx_map"][i] - lo for i in idx], C)
            training.policy_backward(m, ctx, wgt[lo:hi])
            del ctx
            lps.append(lp_c)
        return torch.cat(lps)

    m.zero_grad_buffers()
    lp = chunked(2)
    att = cmask.bool().cuda()
    e_mine, e_ref = (lp - lp_o)[att].abs(), (lp16 - lp_o)[att].abs()
    print(f"(c) logps L={ids.shape[1]}: max|err| ours {e_mine.max():.4f} vs HF-bf16 {e_ref.max():.4f}; mean {e_mine.mean():.5f} vs {e_ref.mean():.5f}")
    assert e_mine.mean().item() <= 1.25 * e_ref.mean().item() + 1e-4
    assert e_mine.max().item() <= 1.25 * e_ref.max().item() + 2e-2
    worst, wname, rw, rb = _grad_report(m, oracle)
    print(f"(c) grads: worst LoRA rel err {worst:.4f} ({wname}); projector dW {rw:.4f} db {rb:.4f}")
    assert worst < 0.03 and rw < 0.03 and rb < 0.03
    # ---- bit-reproducibility of the whole backward (no floating-point atomics anywhere)
    g1 = lora.flat_grad.clone(); pw1 = m._proj_grad_w.clone()
    m.zero_grad_buffers()
    lp_b = chunked(2)
    assert torch.equal(lp_b, lp)
    assert torch.equal(lora.flat_grad, g1) and torch.equal(m._proj_grad_w, pw1), "gradients are not run-to-run reproducible"
    # ---- micro_rows chunking: one-row chunks == two-row chunks (row-separable loss; only the fp32 accumulation order differs)
    m.zero_grad_buffers()
    lp_c = chunked(1)
    assert (lp_c - lp).abs().max().item() < 1e-4                           # forward rows are independent of the chunking
    assert _rel(lora.flat_grad, g1) < 2e-3 and _rel(m._proj_grad_w, pw1) < 2e-3


def test_config_c_rollout_prefix_sharing_greedy_and_eos():
    """Greedy decode at V = 151 936 / d = 2560 with the G = 8 prefix-shared paged KV (28 shared pages at P = 1852): ids vs the oracle's
    greedy loop (margin-aware), graph == eager, and an EOS-terminated rollout (EOS := the token the oracle emits at step 3)."""
    from bioreason_b200.models import DNALLMModel
    from oracle.generate import manual_generate
    from oracle.models import build_oracle, synth_batch
    tc, dc = _cfgs("qwen3-4b")
    oracle = build_oracle(tc, dc, seed=41)
    m = DNALLMModel.from_oracle(oracle)
    G, n = 8, 10
    batch = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=12, same_prompt=True)
    one = dict(input_ids=batch["input_ids"][:1], attention_mask=batch["attention_mask"][:1],
               dna_tokenized={k: v[:2] for k, v in batch["dna_tokenized"].items()}, batch_idx_map=[0, 0])
    oracle = oracle.cuda()                                                                       # the fp32 checker runs on the GPU here
    want, margins = manual_generate(oracle, _cuda_batch(one), max_new_tokens=n, return_margins=True)   # fp32, no EOS
    want, margins = want.cpu().expand(G, -1), margins.cpu().expand(G, -1)
    ids_e, st = m.generate(**batch, max_new_tokens=n, do_sample=False, use_graph=False, return_stats=True)
    ids_g = m.generate(**batch, max_new_tokens=n, do_sample=False, use_graph=True)
    assert st["G"] == G and st["unique_prompts"] == 1 and st["n_shared_pages"] == batch["input_ids"].shape[1] // 64 == 28
    assert torch.equal(ids_e, ids_g), f"graph replay and eager decode disagree: eager {ids_e.tolist()} graph {ids_g.tolist()}"
    assert all(torch.equal(ids_e[0], ids_e[r]) for r in range(G)), "rows of one greedy group must be identical"
    flips = _first_mismatch_ok(ids_e.cpu(), want, margins, tol=0.05)
    print(f"(c) greedy V={tc.vocab_size}: ids {ids_e[0].tolist()} oracle {want[0].tolist()} min margin {margins.min():.3f} near-tie flips {flips}")
    # ---- EOS-terminated: declare the oracle's step-3 token to be EOS; rows stop there, later columns are trimmed / padded
    eos = int(want[0, 3])
    first = int((want[0] == eos).nonzero()[0])
    ids_s = m.generate(**batch, max_new_tokens=n, do_sample=False, eos_token_id=eos, pad_token_id=7)
    if flips == 0:
        assert ids_s.shape[1] == first + 1 and torch.equal(ids_s.cpu(), want[:, :first + 1])
    from bioreason_b200 import ops
    cm = ops.eos_mask(ids_s, eos)
    assert int(cm.sum(1).min()) >= 1 and cm.shape == ids_s.shape


def test_config_b_sft_step_real_widths():
    """Config (b): SFT step, batch 8, 2 x 668-token DNA (4 kb) + 512-token prompt, Qwen3-1.7B widths: CE loss over the assistant span and
    LoRA / projector gradients vs torch autograd on the fp32 oracle."""
    from oracle.models import synth_batch
    tc, dc = _cfgs("qwen3-1.7b")
    oracle, m, lora = _build_pair(tc, dc, seed=51)
    B = 8
    batch = synth_batch(tc, dc, batch=B, n_seq=2, dna_len=668, text_len=[512, 480, 512, 401, 512, 512, 350, 512], seed=14)
    labels = batch["input_ids"].clone()
    labels[batch["attention_mask"] == 0] = -100
    labels[:, : labels.shape[1] - 160] = -100                             # the last 160 tokens are the scored assistant span
    cb = _cuda_batch(batch)
    loss_o = 0.0
    n_valid = (labels[:, 1:] != -100).sum().item()
    for r in range(B):                                                     # row-wise (memory), same global mean
        out = oracle(input_ids=cb["input_ids"][r:r + 1], attention_mask=cb["attention_mask"][r:r + 1],
                     dna_tokenized={k: v[2 * r:2 * r + 2] for k, v in cb["dna_tokenized"].items()}, batch_idx_map=[0, 0])
        lg = out.logits[0, :-1].float()
        tgt = labels[r, 1:].cuda()
        l = torch.nn.functional.cross_entropy(lg, tgt, ignore_index=-100, reduction="sum") / n_valid
        l.backward()
        loss_o += l.item()
    m.zero_grad_buffers()
    loss = m.sft_step(**cb, labels=labels.cuda())
    worst, wname, rw, rb = _grad_report(m, oracle)
    print(f"(b) sft B={B} L={labels.shape[1]}: loss {loss.item():.4f} vs {loss_o:.4f}; worst LoRA rel err {worst:.4f} ({wname}); projector dW {rw:.4f}")
    assert abs(loss.item() - loss_o) < 2e-2 * max(1.0, abs(loss_o))
    assert worst < 0.03 and rw < 0.03 and rb < 0.03


def test_config_e_ragged_kegg_batch_rollout_and_step():
    """Config (e) geometry: ragged KEGG-shape prompts (DNA 666..670 tokens, text 150..250) left-padded, 2 prompts x G = 4: the rollout's
    completions are scored against the oracle (log-probs of the generated tokens) and a full GRPO step runs on them."""
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from oracle.models import synth_batch
    tc, dc = _cfgs("qwen3-4b")
    oracle, m, lora = _build_pair(tc, dc, seed=61)
    G, C = 4, 24
    a = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=[666] * G, text_len=[150] * G, seed=21, same_prompt=True)
    b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=[670] * G, text_len=[250] * G, seed=22, same_prompt=True)
    P = max(a["input_ids"].shape[1], b["input_ids"].shape[1])
    def lpad(x, fill):
        return torch.cat([torch.full((x.shape[0], P - x.shape[1]), fill, dtype=x.dtype), x], 1)
    def rpad(x, fill, S):
        return torch.cat([x, torch.full((x.shape[0], S - x.shape[1]), fill, dtype=x.dtype)], 1)
    S = max(a["dna_tokenized"]["input_ids"].shape[1], b["dna_tokenized"]["input_ids"].shape[1])
    batch = dict(input_ids=torch.cat([lpad(a["input_ids"], tc.pad_token_id), lpad(b["input_ids"], tc.pad_token_id)]),
                 attention_mask=torch.cat([lpad(a["attention_mask"], 0), lpad(b["attention_mask"], 0)]),
                 dna_tokenized=dict(input_ids=torch.cat([rpad(a["dna_tokenized"]["input_ids"], dc.pad_token_id, S), rpad(b["dna_tokenized"]["input_ids"], dc.pad_token_id, S)]),
                                    attention_mask=torch.cat([rpad(a["dna_tokenized"]["attention_mask"], 0, S), rpad(b["dna_tokenized"]["attention_mask"], 0, S)])),
                 batch_idx_map=a["batch_idx_map"] + [i + G for i in b["batch_idx_map"]])
    cfg = DNALLMGRPOConfig(num_generations=G, max_completion_length=C, per_device_train_batch_size=2 * G, learning_rate=1e-4, suppress_eos=True)
    def reward(completion_ids, **kw):
        return (completion_ids % 3 == 0).float().mean(1)
    tr = DNALLMGRPOTrainer(m, [reward], cfg)
    u = torch.rand(C, 2 * G, generator=torch.Generator().manual_seed(1))
    inp = tr._generate_and_score_completions(batch, m, uniforms=u)
    comp = inp["completion_ids"]
    assert comp.shape == (2 * G, C)
    assert not torch.equal(comp[0], comp[G]), "different prompts produced identical rollouts"
    ids = torch.cat([batch["input_ids"].cuda(), comp], 1)
    mask = torch.cat([batch["attention_mask"].cuda(), inp["completion_mask"].long()], 1)
    cb = _cuda_batch(batch)
    # policy log-probs of the sampled tokens (adapters on) and reference-policy log-probs (adapters off) vs the oracle
    with torch.no_grad():
        lp_o = _oracle_logps(oracle, ids, mask, dict(dna_tokenized=cb["dna_tokenized"], batch_idx_map=cb["batch_idx_map"]), C)
    lp = tr._get_per_token_logps(m, ids, mask, keep_last=C, dna_tokenized=cb["dna_tokenized"], batch_idx_map=cb["batch_idx_map"])
    err = (lp - lp_o).abs()
    print(f"(e) ragged P={P} (rows {int(batch['attention_mask'][0].sum())}/{int(batch['attention_mask'][G].sum())} real tokens): |logp err| max {err.max():.4f} mean {err.mean():.5f}")
    assert err.mean().item() < 0.02 and err.max().item() < 0.25
    loss = tr.training_step(inp)
    assert torch.isfinite(loss)
    met = tr.log_metrics()
    assert met["completion_length"] == C and met["kl"] >= 0
