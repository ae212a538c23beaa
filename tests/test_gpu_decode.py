"""GPU parity tests for the rollout kernels (skinny GEMM, paged decode attention, sampler) and generate()."""
import math
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200 import ops
    return ops


@pytest.mark.parametrize("R,N,K", [(8, 2560, 2560), (8, 6144, 2560), (8, 2560, 9728), (3, 512, 256), (16, 1024, 512), (32, 4096, 1024),
                                   (8, 151936, 2560)])
def test_skinny_gemm(ops, R, N, K):
    torch.manual_seed(N + K + R)
    x = torch.randn(R, K).bfloat16().cuda(); w = (torch.randn(N, K) / K ** 0.5).bfloat16().cuda()
    scratch = ops.skinny_scratch(N, "cuda")
    ref = x.float() @ w.float().T
    out = ops.skinny_gemm(x, w, scratch, mode=3)
    torch.testing.assert_close(out, ref, rtol=1e-3, atol=2e-3)
    out2 = ops.skinny_gemm(x, w, scratch, mode=3)                       # scratch must be self-cleaning
    assert torch.equal(out, out2) or (out - out2).abs().max() < 1e-4
    res = torch.randn(R, N).bfloat16().cuda()
    o1 = ops.skinny_gemm(x, w, scratch, mode=1, residual=res)
    torch.testing.assert_close(o1.float(), (ref.bfloat16().float() + res.float()).bfloat16().float(), rtol=2e-2, atol=2e-2)
    o0 = ops.skinny_gemm(x, w, scratch)
    torch.testing.assert_close(o0.float(), ref, rtol=2e-2, atol=2e-2)
    o2 = ops.skinny_gemm(x, w, scratch, mode=2)
    r4 = ref.view(R, N // 16, 2, 8)
    g, u = r4[:, :, 0].reshape(R, N // 2).bfloat16().float(), r4[:, :, 1].reshape(R, N // 2).bfloat16().float()
    torch.testing.assert_close(o2.float(), torch.nn.functional.silu(g).bfloat16().float() * u, rtol=3e-2, atol=2e-2)
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert scratch.view(torch.int32)[n_sms * 32 * 128:].abs().sum().item() == 0          # arrival counters self-reset


def _dense_ref(q, kd, vd, kv_len, Hq, Hkv, D):
    """q [R, Hq*D]; kd/vd [R, T, Hkv*D] dense per-row context; kv_len [R]."""
    R = q.shape[0]
    qf = q.float().view(R, Hq, D)
    rep = Hq // Hkv
    out = torch.zeros(R, Hq, D, device=q.device)
    for r in range(R):
        n = int(kv_len[r])
        k = kd[r, :n].float().view(n, Hkv, D).repeat_interleave(rep, 1)
        v = vd[r, :n].float().view(n, Hkv, D).repeat_interleave(rep, 1)
        s = torch.einsum("hd,nhd->hn", qf[r], k) * D ** -0.5
        out[r] = torch.einsum("hn,nhd->hd", torch.softmax(s, -1), v)
    return out.view(R, Hq * D)


@pytest.mark.parametrize("U,G,Hq,Hkv,plen,gen", [(1, 8, 32, 8, 1848, 37), (2, 4, 16, 8, 200, 70), (3, 1, 4, 2, 90, 5), (1, 8, 4, 2, 50, 1)])
def test_decode_attn_fused_paged_prefix_shared(ops, U, G, Hq, Hkv, plen, gen):
    torch.manual_seed(plen)
    D, PAGE = 128, 64
    R = U * G
    T = plen + gen                                                       # tokens in cache BEFORE this step
    n_shared = (plen // PAGE) if G > 1 else 0
    priv = math.ceil((T + 1 - n_shared * PAGE) / PAGE)
    max_pages = n_shared + priv
    n_pages = U * n_shared + R * priv + 3
    perm = torch.randperm(n_pages)                                       # scattered physical pages
    table = torch.zeros(R, max_pages, dtype=torch.int32); nxt = 0
    for u in range(U):
        sh = perm[nxt:nxt + n_shared]; nxt += n_shared
        for gi in range(G):
            r = u * G + gi
            table[r, :n_shared] = sh.int()
            table[r, n_shared:] = perm[nxt:nxt + priv].int(); nxt += priv
    kd = torch.randn(R, T + 1, Hkv * D).bfloat16(); vd = torch.randn(R, T + 1, Hkv * D).bfloat16()
    for u in range(U):                                                   # the prompt part is identical inside a group
        kd[u * G:(u + 1) * G, :plen] = kd[u * G, :plen].clone(); vd[u * G:(u + 1) * G, :plen] = vd[u * G, :plen].clone()
    kc = torch.zeros(n_pages, Hkv, PAGE, D, dtype=torch.bfloat16); vc = torch.zeros_like(kc)
    for r in range(R):
        for t in range(T):                                               # token T (the new one) is appended by the kernel under test
            pg = table[r, t // PAGE].item()
            kc[pg, :, t % PAGE] = kd[r, t].view(Hkv, D); vc[pg, :, t % PAGE] = vd[r, t].view(Hkv, D)
    kc, vc, table = kc.cuda(), vc.cuda(), table.cuda()
    qkv = torch.randn(R, (Hq + 2 * Hkv) * D).bfloat16().cuda()
    qn = (1 + 0.1 * torch.randn(D)).bfloat16().cuda(); kn = (1 + 0.1 * torch.randn(D)).bfloat16().cuda()
    cur = torch.full((R,), T, dtype=torch.int32).cuda()
    # expected append: K = the prefill-path rope kernel's output at position T, V = the raw projection, both at table[r, T // 64],
    # slot T % 64; every other cache entry stays as it was
    ref_qkv = qkv.clone()
    ops.qk_rope_(ref_qkv, Hq, Hkv, D, cur, 1e6, q_norm_w=qn, k_norm_w=kn, eps=1e-6)
    want_kc, want_vc = kc.clone(), vc.clone()
    for r in range(R):
        pg = table[r, T // PAGE].item()
        want_kc[pg, :, T % PAGE] = ref_qkv[r, Hq * D:(Hq + Hkv) * D].view(Hkv, D)
        want_vc[pg, :, T % PAGE] = qkv[r, (Hq + Hkv) * D:].view(Hkv, D)
        kd[r, T] = ref_qkv[r, Hq * D:(Hq + Hkv) * D].cpu(); vd[r, T] = qkv[r, (Hq + Hkv) * D:].cpu()
    ref = _dense_ref(ref_qkv[:, :Hq * D], kd.cuda(), vd.cuda(), cur + 1, Hq, Hkv, D)
    # one launch (rope + append + both passes + merge) on the RAW projection
    ss = min(8, n_shared) if n_shared else 0
    sp = 2 if n_shared else 8
    ws = ops.decode_fused_workspace(R, Hq, Hkv, D, ss + sp, "cuda")
    out = torch.empty(R, Hq * D, dtype=torch.bfloat16, device="cuda")
    rope = ops.rope_table(T + 2, D, 1e6, "cuda")
    for it in range(3):                                                    # repeated: arrival counters must self-reset
        ops.decode_attn_fused(qkv, qn, kn, kc, vc, table, cur, G, Hq, Hkv, D, n_shared, ss, sp, 1e6, 1e-6, ws, out, rope=rope)
        torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=2e-2)
        assert torch.equal(kc, want_kc) and torch.equal(vc, want_vc), f"rep {it}: appended K/V differ"
    with pytest.raises(RuntimeError, match="cos/sin table"):               # the table is part of the contract (no inline sincos fallback)
        ops.decode_attn_fused(qkv, qn, kn, kc, vc, table, cur, G, Hq, Hkv, D, n_shared, ss, sp, 1e6, 1e-6, ws, out, rope=None)


def _sampler_ref(logits, T, k, p, u):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = logits
    for w in (TemperatureLogitsWarper(T), TopKLogitsWarper(top_k=k), TopPLogitsWarper(top_p=p)):
        s = w(None, s)
    probs = torch.softmax(s, -1)
    cdf = probs.cumsum(-1)
    return (cdf > u[:, None] * cdf[:, -1:]).int().argmax(-1), probs


def test_sampler_matches_hf_warpers(ops):
    torch.manual_seed(0)
    R, V, C = 8, 151936, 6
    tokens = torch.zeros(R, C, dtype=torch.int64, device="cuda"); nxt = torch.zeros(R, dtype=torch.int64, device="cuda")
    fin = torch.zeros(R, dtype=torch.int32, device="cuda"); step = torch.zeros(1, dtype=torch.int32, device="cuda")
    uni = torch.rand(C, R)
    mism = 0
    for s in range(C):
        logits = (torch.randn(R, V) * 2.5)
        logits[0, 5] = logits[0, 77] = logits[0].max() + 1.0              # exact tie at the top
        ref, probs = _sampler_ref(logits, 0.6, 20, 0.95, uni[s])
        step.fill_(s)
        ops.sample_next(logits.cuda(), temperature=0.6, top_k=20, top_p=0.95, do_sample=True, uniforms=uni.cuda(), step=step, max_steps=C,
                        eos_id=-1, pad_id=0, finished=fin, tokens=tokens, next_ids=nxt)
        got = nxt.cpu()
        # the two-stage (chunk candidates -> merge) sampler must make exactly the same choice on the same logits
        nxt2 = torch.zeros_like(nxt); tok2 = torch.zeros_like(tokens)
        ops.sample_next(logits.cuda(), temperature=0.6, top_k=20, top_p=0.95, do_sample=True, uniforms=uni.cuda(), step=step, max_steps=C,
                        eos_id=-1, pad_id=0, finished=fin, tokens=tok2, next_ids=nxt2, workspace=ops.sample_workspace(R, V, "cuda"))
        assert torch.equal(nxt2.cpu(), got)
        assert torch.all(probs.gather(1, got[:, None]) > 0)                # always inside HF's support
        mism += (got != ref).sum().item()
        assert torch.equal(tokens[:, s].cpu(), got)
    assert mism <= 1, f"{mism} draws differ from the HF-warper inverse-CDF"  # fp32 cumsum-order borderline only
    # greedy + EOS/pad bookkeeping
    logits = torch.randn(R, V); logits[3, 123] = 50.0
    fin.zero_(); fin[5] = 1; step.fill_(0)
    ops.sample_next(logits.cuda(), do_sample=False, step=step, max_steps=C, eos_id=123, pad_id=999, finished=fin, tokens=tokens, next_ids=nxt)
    want = logits.argmax(-1); want[5] = 999
    assert torch.equal(nxt.cpu(), want) and fin[3].item() == 1 and fin[5].item() == 1 and fin[0].item() == 0
    fin.zero_(); fin[5] = 1
    ops.sample_next(logits.cuda(), do_sample=False, step=step, max_steps=C, eos_id=123, pad_id=999, finished=fin, tokens=tokens, next_ids=nxt,
                    workspace=ops.sample_workspace(R, V, "cuda"))
    assert torch.equal(nxt.cpu(), want) and fin[3].item() == 1


@pytest.mark.parametrize("kind", ["narrow", "constant", "masked", "ties", "wide"])
def test_sampler_two_stage_degenerate_distributions(ops, kind):
    """The two-stage sampler picks its candidates from a histogram over the distance to the maximum and falls back to an exact radix
    select when that is not selective (many values within 1/32 of the k-th).  Whatever path runs, the draw must equal the single-stage
    exact sampler's and HF's warpers: logits with a tiny spread, constant rows, rows that are -inf except a few entries, massive ties."""
    torch.manual_seed(11)
    R, V, C = 8, 151936, 3
    g = torch.Generator().manual_seed(5)
    if kind == "narrow":
        logits = torch.randn(R, V, generator=g) * 1e-3                      # everything within one bin of the maximum
    elif kind == "constant":
        logits = torch.zeros(R, V)                                           # 151 911 exact ties below 25 distinct small bumps
        logits[:, torch.arange(25) * 6007 + 13] = torch.arange(1, 26).float() * 1e-4
    elif kind == "masked":
        logits = torch.full((R, V), float("-inf"))
        idx = torch.randint(0, V, (R, 40), generator=g)
        logits.scatter_(1, idx, torch.randn(R, 40, generator=g) * 3)
    elif kind == "ties":
        logits = torch.randn(R, V, generator=g).mul(4).round().div(4)        # quantised: hundreds of exact ties at every level
    else:
        logits = torch.randn(R, V, generator=g) * 30                        # far beyond the 64-unit histogram range
    uni = torch.rand(C, R, generator=g)
    fin = torch.zeros(R, dtype=torch.int32, device="cuda"); step = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = ops.sample_workspace(R, V, "cuda")
    for s_ in range(C):
        step.fill_(s_)
        a = torch.zeros(R, dtype=torch.int64, device="cuda"); b = torch.zeros_like(a)
        kw = dict(temperature=0.6, top_k=20, top_p=0.95, do_sample=True, uniforms=uni.cuda(), step=step, max_steps=C, eos_id=-1, pad_id=0, finished=fin)
        ops.sample_next(logits.cuda(), next_ids=a, **kw)
        ops.sample_next(logits.cuda(), next_ids=b, workspace=ws, **kw)
        assert torch.equal(a.cpu(), b.cpu()), kind
        if kind not in ("constant", "ties", "narrow"):                       # HF keeps EVERY tie of the k-th value; same support here
            ref, probs = _sampler_ref(logits, 0.6, 20, 0.95, uni[s_])
            assert torch.all(probs.gather(1, a.cpu()[:, None]) > 0)
        # greedy
        ops.sample_next(logits.cuda(), do_sample=False, step=step, max_steps=C, eos_id=-1, pad_id=0, finished=fin, next_ids=b, workspace=ws)
        assert torch.equal(b.cpu(), logits.argmax(-1)) or kind in ("ties", "constant", "narrow")
        if kind in ("ties", "constant"):                                     # ties: the smallest token id among the maxima
            mx = logits.max(-1, keepdim=True).values
            first = (logits == mx).int().argmax(-1)
            assert torch.equal(b.cpu(), first)


def _first_mismatch_ok(got, want, margins, tol):
    """Greedy ids must be bit-exact except where the oracle's own top-2 margin is below the bf16 noise floor; after such
    a near-tie flip the continuations legitimately diverge, so comparison of that row stops there."""
    n_flip = 0
    for r in range(want.shape[0]):
        for t in range(min(got.shape[1], want.shape[1])):
            if got[r, t] != want[r, t]:
                assert margins[r, t] < tol, f"row {r} step {t}: ids differ with oracle margin {margins[r, t]:.4f}"
                n_flip += 1
                break
    return n_flip


def test_generate_greedy_tiny_golden(golden, tiny_oracle):
    from bioreason_b200.models import DNALLMModel
    from oracle.generate import manual_generate
    m = DNALLMModel.from_oracle(tiny_oracle)
    D = golden["D"]; cfg = tiny_oracle.text_config
    for key_b, key_ids, n in (("batch", "greedy", 12), ("ragged_batch", "ragged_greedy", 8)):
        _, margins = manual_generate(tiny_oracle, D[key_b], max_new_tokens=n, eos_token_id=cfg.eos_token_id,
                                     pad_token_id=cfg.pad_token_id, return_margins=True)
        for use_graph in (False, True):
            ids, st = m.generate(**D[key_b], max_new_tokens=n, do_sample=False, pad_token_id=cfg.pad_token_id,
                                 eos_token_id=cfg.eos_token_id, use_graph=use_graph, return_stats=True)
            flips = _first_mismatch_ok(ids.cpu(), D[key_ids], margins, tol=0.02)
            print(key_b, "graph" if use_graph else "eager", st, "near-tie flips:", flips, ids.cpu().tolist()[0])
            assert ids.shape[1] <= n
    assert st["G"] == 1
    _, st = m.generate(**D["batch"], max_new_tokens=4, do_sample=False, return_stats=True)
    assert st["G"] == 4 and st["unique_prompts"] == 1                      # the G-replicated prompt is prefilled once


def test_generate_sampled_small_vs_oracle():
    """Sampled rollout with supplied uniforms vs the oracle's HF-warper loop, prompts long enough to share pages."""
    from bioreason_b200.configs import text_config, dna_config
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle, synth_batch
    from oracle.generate import manual_generate
    tc, dc = text_config("small"), dna_config("small")
    oracle = build_oracle(tc, dc, seed=5)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=50, text_len=60, seed=8, same_prompt=True)
    C = 10
    u = torch.rand(C, 4, generator=torch.Generator().manual_seed(1))
    want = manual_generate(oracle, batch, max_new_tokens=C, do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u)
    m = DNALLMModel.from_oracle(oracle)
    got, st = m.generate(**batch, max_new_tokens=C, do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u, return_stats=True)
    got = got.cpu()
    assert st["G"] == 4 and st["n_shared_pages"] == (60 + 2 + 2 * 50) // 64
    # (1) replayable: same uniforms -> same rollout; different uniforms -> different rollout
    got2 = m.generate(**batch, max_new_tokens=C, do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u).cpu()
    assert torch.equal(got, got2)
    u2 = torch.rand(C, 4, generator=torch.Generator().manual_seed(2))
    assert not torch.equal(got, m.generate(**batch, max_new_tokens=C, do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u2).cpu())
    assert len({tuple(r.tolist()) for r in got}) == 4                      # the G samples of the shared prompt differ
    # (2) teacher-forced support check: every sampled token must be (within bf16 noise of) the oracle's top-k set for
    #     the prefix the CUDA path actually generated.  (Token-for-token equality with the fp32 oracle is ill-conditioned
    #     for a random-init model: the 20th/21st logits differ by less than bf16 noise, and one membership swap shifts
    #     the whole inverse CDF.  Exact draw parity is asserted on identical logits in test_sampler_matches_hf_warpers.)
    full = dict(batch)
    full["input_ids"] = torch.cat([batch["input_ids"], got], 1)
    full["attention_mask"] = torch.cat([batch["attention_mask"], torch.ones_like(got)], 1)
    with torch.no_grad():
        logits = oracle(**full).logits.float()
    P = batch["input_ids"].shape[1]
    worst = 0
    for t in range(C):
        step_logits = logits[:, P - 1 + t]
        rank = (step_logits > step_logits.gather(1, got[:, t:t + 1])).sum(1)      # 0 = argmax
        worst = max(worst, int(rank.max()))
    agree = sum(int((got[r] == want[r]).int().cumprod(0).sum()) for r in range(4))
    print("sampled: worst oracle rank of a drawn token", worst, "| prefix agreement with the fp32-oracle draw:", agree, "/", 4 * C)
    assert worst < 20 + 4


@pytest.mark.parametrize("R,d,F,nqkv,V", [(8, 2560, 9728, 6144, 4096), (8, 256, 512, 1024, 1024), (3, 512, 1536, 1536, 4096)])
def test_skinny_layer_sequence_is_reproducible(ops, R, d, F, nqkv, V):
    """The decode layer's GEMM sequence o_proj -> gate/up -> down_proj -> next qkv | lm_head, launched one by one on ONE scratch
    buffer, repeated: every run is bit-identical (the stream-K reduction is fixed-order and the arrival counters self-reset)."""
    torch.manual_seed(d + F)
    bf = torch.bfloat16
    mk = lambda *s_: (torch.randn(*s_, device="cuda") * (1.0 / s_[-1] ** 0.5)).to(bf)
    HqD = d if d < 2560 else 4096
    w_o, w_gu, w_down, w_qkv, w_lm = mk(d, HqD), mk(2 * F, d), mk(d, F), mk(nqkv, d), mk(V, d)
    attn = torch.randn(R, HqD, device="cuda").to(bf); h0 = torch.randn(R, d, device="cuda").to(bf)
    n_part = ((d + 127) // 128) * 4
    scratch = ops.skinny_scratch(max(V, 2 * F), "cuda")

    def layer():
        h = h0.clone(); ssa = torch.zeros(n_part, 32, device="cuda"); ssb = torch.zeros(n_part, 32, device="cuda")
        x2 = ops.skinny_gemm(attn, w_o, scratch, mode=1, residual=h, sumsq_out=ssb)
        act = ops.skinny_gemm(x2, w_gu, scratch, mode=2, sumsq_in=ssb, sumsq_in_n=n_part, eps=1e-6)
        hn = ops.skinny_gemm(act, w_down, scratch, mode=1, residual=x2, sumsq_out=ssa)
        qkv = ops.skinny_gemm(hn, w_qkv, scratch, sumsq_in=ssa, sumsq_in_n=n_part, eps=1e-6)
        lg = ops.skinny_gemm(hn, w_lm, scratch, mode=3, sumsq_in=ssa, sumsq_in_n=n_part, eps=1e-6)
        return x2, act, hn, qkv, lg
    first = layer()
    for rep in range(1, 3):
        again = layer()
        for name, a, b in zip(("x2", "act", "h", "qkv", "lm_head"), first, again):
            assert torch.equal(a, b), f"rep {rep}: {name} differs"
    # sanity of the first GEMM against fp32 math
    ref_x2 = (attn.float() @ w_o.float().T).bfloat16().float() + h0.float()
    torch.testing.assert_close(first[0].float(), ref_x2.bfloat16().float(), rtol=2e-2, atol=2e-2)


def test_generate_eos_and_multi_group(golden, tiny_oracle):
    """EOS bookkeeping end to end (finished rows emit pad, output trimmed to the longest row, HF generation/utils.py:2796-2797) and a
    batch of two different prompt groups (U=2, G=2) against the oracle loop."""
    from bioreason_b200.configs import text_config, dna_config
    from bioreason_b200.models import DNALLMModel
    from oracle.generate import manual_generate
    from oracle.models import synth_batch
    m = DNALLMModel.from_oracle(tiny_oracle)
    D = golden["D"]; cfg = tiny_oracle.text_config
    # make the token greedy decoding emits at step 4 the EOS: every row of the replicated prompt stops there
    eos = int(D["greedy"][0, 4])
    want = manual_generate(tiny_oracle, D["batch"], max_new_tokens=12, eos_token_id=eos, pad_token_id=cfg.pad_token_id)
    got = m.generate(**D["batch"], max_new_tokens=12, do_sample=False, eos_token_id=eos, pad_token_id=cfg.pad_token_id).cpu()
    assert got.shape == want.shape == (4, 5) and torch.equal(got, want)
    # ragged: rows finish at different steps -> pads after EOS, trimmed to the longest
    rb = D["ragged_batch"]
    base = manual_generate(tiny_oracle, rb, max_new_tokens=8)
    eos = int(base[1, 2])
    want, margins = manual_generate(tiny_oracle, rb, max_new_tokens=8, eos_token_id=eos, pad_token_id=cfg.pad_token_id, return_margins=True)
    got = m.generate(**rb, max_new_tokens=8, do_sample=False, eos_token_id=eos, pad_token_id=cfg.pad_token_id).cpu()
    assert got.shape[1] == want.shape[1]
    _first_mismatch_ok(got, want, margins, tol=0.02)
    # two prompt groups of G=2 (different lengths): grouping is detected, both groups prefilled once
    tc, dc = tiny_oracle.text_config, tiny_oracle.dna_config
    a = synth_batch(tc, dc, batch=2, n_seq=1, dna_len=9, text_len=40, seed=21, same_prompt=True)
    b = synth_batch(tc, dc, batch=2, n_seq=1, dna_len=9, text_len=70, seed=22, same_prompt=True)
    L = max(a["input_ids"].shape[1], b["input_ids"].shape[1])
    def lpad(x, fill):
        return torch.cat([torch.full((x.shape[0], L - x.shape[1]), fill, dtype=x.dtype), x], 1)
    mix = dict(input_ids=torch.cat([lpad(a["input_ids"], tc.pad_token_id), lpad(b["input_ids"], tc.pad_token_id)]),
               attention_mask=torch.cat([lpad(a["attention_mask"], 0), lpad(b["attention_mask"], 0)]),
               dna_tokenized={k: torch.cat([a["dna_tokenized"][k], b["dna_tokenized"][k]]) for k in ("input_ids", "attention_mask")},
               batch_idx_map=[0, 1, 2, 3])
    want, margins = manual_generate(tiny_oracle, mix, max_new_tokens=6, return_margins=True)
    got, st = m.generate(**mix, max_new_tokens=6, do_sample=False, return_stats=True)
    assert st["G"] == 2 and st["unique_prompts"] == 2
    _first_mismatch_ok(got.cpu(), want, margins, tol=0.02)


def test_decode_capture_is_safe_from_the_cyclic_collector(golden, tiny_oracle, monkeypatch):
    """A model and its rollout engine reference each other, so a dropped model's captured decode graph lives until Python's cyclic
    collector runs, and destroying a graph while a stream captures invalidates that capture.  generate() must free such garbage
    before it captures and keep the collector off during the capture (a collection there once broke the next rollout, depending on
    how many objects earlier tests had allocated)."""
    import gc
    import weakref
    from bioreason_b200.models import DNALLMModel
    D = golden["D"]
    old = DNALLMModel.from_oracle(tiny_oracle)
    old.generate(**D["batch"], max_new_tokens=12, do_sample=False)
    assert old._rollout._cached, "the first rollout captured a decode graph"
    probe = weakref.ref(old._rollout)
    was_enabled = gc.isenabled()
    gc.disable()
    try:
        del old
        assert probe() is not None, "the model / engine cycle keeps the captured graph alive after the model is dropped"
    finally:
        if was_enabled:
            gc.enable()
    seen = []
    enter = torch.cuda.graph.__enter__

    def spy(self):
        seen.append((gc.isenabled(), probe() is None))
        return enter(self)
    monkeypatch.setattr(torch.cuda.graph, "__enter__", spy)
    m = DNALLMModel.from_oracle(tiny_oracle)
    got = m.generate(**D["batch"], max_new_tokens=12, do_sample=False).cpu()
    assert seen == [(False, True)], "capture must start with the collector off and the dropped engine (and its graph) freed"
    assert gc.isenabled() == was_enabled
    assert torch.equal(got, m.generate(**D["batch"], max_new_tokens=12, do_sample=False, use_graph=False).cpu())


def test_generate_ignores_recycled_allocator_garbage(golden, tiny_oracle):
    """Buffers of a rollout come from torch's caching allocator, i.e. they may hold anything -- including NaN bit patterns -- that an
    earlier tensor left behind.  Masked positions are multiplied by exact-zero probabilities, which is only harmless for finite
    operands: the paged KV cache is zero-filled once, every other buffer is fully written before it is read.  (Found by running the
    config (c) rollout test after the backward tests in one process: eager and graph rollouts disagreed.)"""
    from bioreason_b200.models import DNALLMModel
    D = golden["D"]
    clean = DNALLMModel.from_oracle(tiny_oracle).generate(**D["batch"], max_new_tokens=12, do_sample=False).cpu()
    for rep in range(2):
        junk = [torch.full((n,), float("nan"), device="cuda", dtype=torch.bfloat16) for n in (1 << 18, 1 << 20, 1 << 22, 1 << 24)]
        junk += [torch.full((n,), float("inf"), device="cuda", dtype=torch.float32) for n in (1 << 18, 1 << 20, 1 << 22)]
        del junk                                                             # back to the allocator's free lists, contents intact
        m = DNALLMModel.from_oracle(tiny_oracle)                            # fresh rollout caches -> recycled blocks
        for use_graph in (False, True):
            got = m.generate(**D["batch"], max_new_tokens=12, do_sample=False, use_graph=use_graph).cpu()
            assert torch.equal(got, clean), f"rep {rep} graph={use_graph}"
