"""Weight-only FP8 (e4m3) rollout decode: the per-row quantizer, the FP8 instantiation of the decode GEMM, the rollout plumbing and
the trainer flag.  The e4m3 layout is private to the two kernels, so the codes are read back through the GEMM (one-hot X rows)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decode_ref as dr  # noqa: E402

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
# (N, K) of the four decode matrices: qkv, o, gate/up (2F), down
QWEN3_4B = [(6144, 2560), (2560, 4096), (19456, 2560), (2560, 9728)]
QWEN3_1P7B = [(4096, 2048), (2048, 2048), (12288, 2048), (2048, 6144)]
STREAMK_SPLIT = (256, 4096)          # 2 feature tiles x 64 k blocks = 128 units < one per SM: every tile spans many CTAs


@pytest.fixture(scope="module")
def ops():
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def scratch(ops):
    return ops.skinny_scratch(2 * 19456, "cuda")


def ref_quant(w):
    """The definition: scale = amax|row| / 448 (1 for a zero row), codes = RNE(w / scale) in e4m3fn.  Both divisions are correctly
    rounded: the divisor is a tensor, because torch on CUDA turns a division by a Python scalar into a multiplication by its
    reciprocal, which differs in the last bit for some amax."""
    amax = w.float().abs().amax(1)
    scale = torch.where(amax > 0, amax / torch.full_like(amax, 448.0), torch.ones_like(amax))
    return (w.float() / scale[:, None]).to(E4M3), scale


def dequant(q8, scale):
    return q8.float() * scale[:, None]


def read_back(ops, fw, scratch):
    """dequant(Q) as the FP8 GEMM sees it: X = one-hot rows (mode 3, fp32 out, no norm) give column k of scale * codes exactly."""
    N, K = fw.shape
    out = torch.empty(N, K, device="cuda")
    for k0 in range(0, K, 32):
        R = min(32, K - k0)
        x = torch.zeros(R, K, device="cuda", dtype=torch.bfloat16)
        x[torch.arange(R), k0 + torch.arange(R)] = 1
        out[:, k0:k0 + R] = ops.skinny_gemm(x, fw, scratch, mode=3).T
    return out


def special_matrix(N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn(N, K, device="cuda", generator=g) * 0.02
    w[0] = 0                                                               # all-zero row: scale 1, all codes 0
    w[1] = 0; w[1, K // 3] = -0.37                                         # one non-zero entry: codes 0 and -448
    w[2] = torch.rand(K, device="cuda", generator=g) * 2.0 ** -6 * torch.sign(torch.randn(K, device="cuda", generator=g))
    w[2, 0] = 448.0                                                        # scale 1: the rest falls in e4m3's subnormal range
    w[3, :4] = torch.tensor([448.0, -448.0, 440.0, -436.0], device="cuda") * 2.0 ** -5   # values that round exactly to +-448
    return w.bfloat16()


@pytest.mark.parametrize("N,K", QWEN3_4B + QWEN3_1P7B)
def test_quantizer_bit_exact(ops, scratch, N, K):
    w = special_matrix(N, K, seed=N + K)
    fw = ops.quantize_rows_e4m3(w)
    q_ref, s_ref = ref_quant(w)
    assert torch.equal(fw.scale, s_ref)
    assert s_ref[0].item() == 1.0
    got = read_back(ops, fw, scratch)
    want = dequant(q_ref, s_ref)
    assert torch.equal(got, want), f"{(got != want).sum().item()} codes differ"
    assert not torch.isnan(q_ref.float()).any()
    assert (q_ref.float()[3, :2].abs() == 448).all() and (q_ref.float()[2].abs() < 2.0 ** -6).sum() > K // 2


def test_layout_and_conversion_all_codes(ops, scratch):
    """A matrix whose rows hold all 254 non-NaN e4m3 codes, times power-of-two row scales: the quantizer recovers the codes and the
    GEMM's e4m3 -> bf16 register conversion returns every one of them exactly."""
    codes = torch.tensor([b for b in range(256) if b not in (0x7F, 0xFF)], dtype=torch.uint8)
    vals = codes.view(E4M3).float()
    N, K = 256, 512
    g = torch.Generator().manual_seed(0)
    rows = []
    for n in range(N):
        row = torch.cat([vals[torch.randperm(254, generator=g)], vals[torch.randperm(254, generator=g)], torch.full((4,), 448.0)])
        rows.append(row * 2.0 ** ((n % 24) - 16))
    w = torch.stack(rows).cuda().bfloat16()
    assert torch.equal(w.float().cpu(), torch.stack(rows))                  # e4m3 values x 2^e are bf16-exact
    fw = ops.quantize_rows_e4m3(w)
    assert torch.equal(fw.scale.cpu(), torch.tensor([2.0 ** ((n % 24) - 16) for n in range(N)]))
    assert torch.equal(read_back(ops, fw, scratch), w.float())


# ------------------------------------------------------------------ FP8 GEMM against float64
def _fp64_case(ops, scratch, R, N, K, mode, norm, seed, wrong=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).bfloat16()
    fw = ops.quantize_rows_e4m3(w)
    q, s = ref_quant(w)
    wd = dequant(q, s).double()
    if wrong == "per_column":
        wd = q.double() * s.double()[torch.arange(K, device="cuda") % N][None, :]
    elif wrong == "up_gate_scale":                                          # the up features (lanes 8-15 of each 16) use the gate's scale
        idx = torch.arange(N, device="cuda")
        src = torch.where((idx & 8) != 0, idx - 8, idx)
        wd = q.double() * s.double()[src][:, None]
    x = torch.randn(R, K, device="cuda", generator=g).bfloat16()
    res = torch.randn(R, N, device="cuda", generator=g).bfloat16() if mode == 1 else None
    n_part = 7
    ssq = (torch.rand(n_part, 32, device="cuda", generator=g) * K / n_part + 0.1) if norm else None
    eps = 1e-6
    want_ssq_out = norm and mode <= 1
    ssq_out = torch.full((((N + 127) // 128) * 4, 32), float("nan"), device="cuda") if want_ssq_out else None
    got = ops.skinny_gemm(x, fw, scratch, mode=mode, residual=res, sumsq_in=ssq, sumsq_in_n=n_part if norm else 1, sumsq_out=ssq_out,
                          eps=eps).double()
    ref, bound = dr.skinny_ref(x, wd, mode, residual=res, sumsq_in=ssq, sumsq_in_n=n_part if norm else 1, eps=eps)
    err = (got - ref).abs()
    if wrong is None and want_ssq_out:
        sref, sbound = dr.sumsq_out_ref(got, N)                             # of the kernel's own bf16 outputs
        assert dr.worst_ratio(ssq_out[:, :R], sref, sbound) <= 1.0
    return (err / bound.clamp_min(1e-30)).max().item(), (err > bound).sum().item()


FP64_SHAPES = QWEN3_4B + QWEN3_1P7B + [STREAMK_SPLIT]


@pytest.mark.parametrize("N,K", FP64_SHAPES)
def test_fp8_gemm_vs_fp64(ops, scratch, N, K):
    worst = {}
    for i, R in enumerate((1, 3, 8, 9, 16, 17, 32)):
        for mode in (0, 1, 2, 3):
            norm = (i + mode) % 2 == 0
            ratio, n_bad = _fp64_case(ops, scratch, R, N, K, mode, norm, seed=R * 131 + mode * 7 + N)
            worst[(R, mode, norm)] = ratio
            assert n_bad == 0, f"R={R} mode={mode} norm={norm}: {n_bad} outputs beyond the bound (worst err/bound {ratio:.3f})"
    print(f"{N}x{K}: worst err/bound {max(worst.values()):.4f} at {max(worst, key=worst.get)}")


def test_fp64_bound_rejects_wrong_scales(ops, scratch):
    """The bound is tight enough to see a scale applied per column, or the up feature scaled with its gate's scale."""
    r_col, _ = _fp64_case(ops, scratch, 8, 2560, 4096, 3, False, seed=1, wrong="per_column")
    r_gate, _ = _fp64_case(ops, scratch, 8, 19456, 2560, 2, False, seed=2, wrong="up_gate_scale")
    print(f"wrong references: per-column scale err/bound {r_col:.1f}, up-with-gate-scale {r_gate:.1f}")
    assert r_col > 1 and r_gate > 1


def test_fp8_equals_bf16_on_grid_weights(ops, scratch):
    """Weights already on the per-row e4m3 grid with power-of-two scales: the FP8 GEMM computes the bf16 GEMM's products and sums,
    so every mode returns the same bits (what the end-to-end rollout comparison below rests on)."""
    N, K, R = 2048, 2560, 8
    w = grid_matrix(N, K, seed=3)
    fw = ops.quantize_rows_e4m3(w)
    x = torch.randn(R, K, device="cuda").bfloat16()
    res = torch.randn(R, N, device="cuda").bfloat16()
    ssq = torch.rand(4, 32, device="cuda") * K
    for mode in (0, 1, 2, 3):
        kw = dict(mode=mode, residual=res if mode == 1 else None, sumsq_in=ssq, sumsq_in_n=4, eps=1e-6)
        assert torch.equal(ops.skinny_gemm(x, fw, scratch, **kw), ops.skinny_gemm(x, w, scratch, **kw)), mode


def test_fp8_layer_sequence_is_reproducible(ops, scratch):
    """The decode layer's GEMM sequence on FP8 weights and one scratch buffer, repeated: bit-identical."""
    torch.manual_seed(7)
    R, d, F, nqkv, HqD = 8, 2560, 9728, 6144, 4096
    mk = lambda *s_: ops.quantize_rows_e4m3((torch.randn(*s_, device="cuda") * s_[-1] ** -0.5).bfloat16())
    w_o, w_gu, w_down, w_qkv = mk(d, HqD), mk(2 * F, d), mk(d, F), mk(nqkv, d)
    attn = torch.randn(R, HqD, device="cuda").bfloat16(); h0 = torch.randn(R, d, device="cuda").bfloat16()
    n_part = ((d + 127) // 128) * 4

    def layer():
        h = h0.clone(); ssa = torch.zeros(n_part, 32, device="cuda"); ssb = torch.zeros(n_part, 32, device="cuda")
        x2 = ops.skinny_gemm(attn, w_o, scratch, mode=1, residual=h, sumsq_out=ssb)
        act = ops.skinny_gemm(x2, w_gu, scratch, mode=2, sumsq_in=ssb, sumsq_in_n=n_part, eps=1e-6)
        hn = ops.skinny_gemm(act, w_down, scratch, mode=1, residual=x2, sumsq_out=ssa)
        qkv = ops.skinny_gemm(hn, w_qkv, scratch, sumsq_in=ssa, sumsq_in_n=n_part, eps=1e-6)
        return x2, act, hn, qkv, ssa, ssb
    first = layer()
    for _ in range(2):
        for a, b in zip(first, layer()):
            assert torch.equal(a, b)


def test_refuses_unsupported_shapes(ops, scratch):
    with pytest.raises(RuntimeError, match="multiple of 16"):
        ops.quantize_rows_e4m3(torch.zeros(128, 24, device="cuda", dtype=torch.bfloat16))
    fw = ops.fp8_weight_empty(128, 24, "cuda")
    with pytest.raises(RuntimeError, match="multiple of 16"):
        ops.skinny_gemm(torch.zeros(2, 24, device="cuda", dtype=torch.bfloat16), fw, scratch)


# ------------------------------------------------------------------ rollout end to end
def grid_matrix(N, K, seed):
    """bf16 [N, K] on the per-row e4m3 grid: power-of-two row scales and one +-448 * scale entry per row."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = 2.0 ** torch.randint(-14, -8, (N, 1), device="cuda", generator=g).float()
    q = (torch.randn(N, K, device="cuda", generator=g) * 60).clamp(-448, 448).to(E4M3).float()
    q[torch.arange(N), torch.randint(0, K, (N,), device="cuda", generator=g)] = 448.0
    return (q * s).bfloat16()


def grid_exact_oracle(size, seed):
    """An oracle model whose decoder linears lie on the per-row e4m3 grid and whose ln1 / ln2 gains are 1: the folded decode
    matrices are grid-exact, so the FP8 rollout computes the same products as the bf16 one."""
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


@pytest.mark.parametrize("size", ["tiny", "small"])
def test_rollout_fp8_equals_bf16_on_grid_weights(size):
    from bioreason_b200.models import DNALLMModel
    from oracle.models import synth_batch
    oracle, tc, dc = grid_exact_oracle(size, seed=11)
    bf = DNALLMModel.from_oracle(oracle)
    f8 = DNALLMModel.from_oracle(oracle)
    f8.set_fp8_rollout(True)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=50, text_len=60, seed=8, same_prompt=True)
    two = [synth_batch(tc, dc, batch=2, n_seq=1, dna_len=9, text_len=n, seed=s, same_prompt=True) for n, s in ((40, 21), (70, 22))]
    C = 12
    for use_graph in (False, True):
        want = bf.generate(**batch, max_new_tokens=C, do_sample=False, use_graph=use_graph).cpu()
        got = f8.generate(**batch, max_new_tokens=C, do_sample=False, use_graph=use_graph).cpu()
        assert torch.equal(got, want), use_graph
    from bioreason_b200.ops import Fp8Weight
    assert isinstance(f8._rollout_dec.layers[0].w_gu, Fp8Weight)
    # sampled, with supplied uniforms: replayable and the same draws as bf16
    u = torch.rand(C, 4, generator=torch.Generator().manual_seed(1))
    kw = dict(max_new_tokens=C, do_sample=True, temperature=0.6, top_k=20, top_p=0.95, uniforms=u)
    a = f8.generate(**batch, **kw).cpu()
    assert torch.equal(a, f8.generate(**batch, **kw).cpu())
    assert torch.equal(a, bf.generate(**batch, **kw).cpu())
    # other prompt lengths, and EOS: the token greedy decoding emits at step 3 ends every row there
    for b2 in two:
        ids = bf.generate(**b2, max_new_tokens=8, do_sample=False).cpu()
        eos = int(ids[0, 3])
        for use_graph in (False, True):
            w_ = bf.generate(**b2, max_new_tokens=8, do_sample=False, eos_token_id=eos, pad_token_id=0, use_graph=use_graph).cpu()
            g_ = f8.generate(**b2, max_new_tokens=8, do_sample=False, eos_token_id=eos, pad_token_id=0, use_graph=use_graph).cpu()
            assert torch.equal(g_, w_)


def test_toggle_off_restores_bf16_rollout():
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config("small"), dna_config("small")
    oracle = build_oracle(tc, dc, seed=5)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=50, text_len=60, seed=8, same_prompt=True)
    never = DNALLMModel.from_oracle(oracle)
    m = DNALLMModel.from_oracle(oracle)
    want = never.generate(**batch, max_new_tokens=10, do_sample=False).cpu()
    m.set_fp8_rollout(True)
    f8 = m.generate(**batch, max_new_tokens=10, do_sample=False).cpu()
    m.set_fp8_rollout(False)
    assert torch.equal(m.generate(**batch, max_new_tokens=10, do_sample=False).cpu(), want)
    print("random-init small model, greedy: FP8 and bf16 ids agree on", int((f8 == want).int().cumprod(1).sum()), "of", want.numel())


# ------------------------------------------------------------------ trainer
def _token_reward(completion_ids, **kw):
    return (completion_ids % 7 == 0).float().sum(1) - 0.1 * (completion_ids % 5 == 0).float().sum(1)


@pytest.mark.parametrize("share", [False, True])
def test_training_step_fp8_rollout(ops, scratch, share):
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.lora import build_rollout_weights
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.trainer import DNALLMGRPOConfig, DNALLMGRPOTrainer
    from oracle.models import build_oracle, synth_batch
    tc, dc = text_config("tiny"), dna_config("tiny")
    oracle = build_oracle(tc, dc, seed=21)
    batch = synth_batch(tc, dc, batch=4, n_seq=2, dna_len=10, text_len=18, seed=14, same_prompt=True)
    m = DNALLMModel.from_oracle(oracle)
    cfg = DNALLMGRPOConfig(num_generations=4, max_completion_length=6, per_device_train_batch_size=4, learning_rate=1e-2, lora_r=16,
                           lora_alpha=32.0, num_iterations=2, fp8_rollout=True, share_prompt_prefix=share)
    tr = DNALLMGRPOTrainer(m, [_token_reward], cfg)
    assert m._fp8_rollout
    for _ in range(2):
        assert torch.isfinite(tr.training_step(batch))
    # the FP8 rollout weights are the reference quantizer applied to the merged, folded weights of the updated adapters
    want = build_rollout_weights(m._dec, m._lora)
    for Lf, Lb in zip(m._rollout_dec.layers, want.layers):
        for name in ("w_qkv", "w_o", "w_gu", "w_down"):
            q, s = ref_quant(getattr(Lb, name))
            fw = getattr(Lf, name)
            assert torch.equal(fw.scale, s), name
            assert torch.equal(read_back(ops, fw, scratch), dequant(q, s)), name
    assert torch.equal(m._rollout_dec.lm_head, want.lm_head)
    assert any(not torch.equal(p, torch.zeros_like(p)) for p in m._lora.params[1::2])    # the adapters moved: B != 0
