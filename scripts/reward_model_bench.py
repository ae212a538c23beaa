"""Cost of scoring GRPO completions with a sequence-classification reward model on the CUDA decoder.

  - pass: CUDA-event time of one RewardModel call (embed_gather -> decoder_forward -> br_seqcls_score) against HF's bf16 sdpa forward
    of the same model, for Qwen3-1.7B- and Qwen3-4B-shaped reward models (random init) at B = 8, L in {512, 2048}, right padded with
    ragged lengths; the two paths alternate call by call after a warm-up;
  - config (c) (Qwen3-4B policy, random init, LoRA r = 32, 1 prompt x G = 8, P = 1852, C = 512, EOS suppressed): training_step wall
    time with a token-level reward function only, and with a Qwen3-1.7B-shaped reward model added, the two trainers alternating step
    by step on one policy in one process after a warm-up step each.
Prints one JSON object with the card name and power limit it was measured on.

    python scripts/reward_model_bench.py [--reps 5] [--no-train] [--out FILE]
"""
import argparse, copy, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

N_WORDS = 50000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                                  # the numbers stay usable without it
        return f"unknown ({e})"


def median(v):
    return sorted(v)[len(v) // 2]


def timed_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def reward_model(name, seed=0):
    from transformers import Qwen3ForSequenceClassification
    from bioreason_b200.configs import text_config
    cfg = text_config(name)
    cfg.num_labels = 1
    torch.manual_seed(seed)
    with torch.device("cuda"):
        return Qwen3ForSequenceClassification(cfg).to(torch.bfloat16).eval()


def word_tokenizer():
    """Word-level tokenizer over w0 .. w{N_WORDS - 1} (+ [UNK], <eos>, <pad>), built in memory."""
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    vocab = {"[UNK]": 0, "<eos>": 1, "<pad>": 2}
    vocab.update({f"w{i}": 3 + i for i in range(N_WORDS)})
    tk = Tokenizer(models.WordLevel(vocab=vocab, unk_token="[UNK]"))
    tk.pre_tokenizer = pre_tokenizers.Whitespace()
    return PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="[UNK]", eos_token="<eos>", pad_token="<pad>")


class WordTok:
    """Policy processing class: token t decodes to the word w<t mod N_WORDS>."""
    eos_token_id = pad_token_id = None

    def batch_decode(self, ids, skip_special_tokens=False):
        return [" ".join(f"w{t % N_WORDS}" for t in row) for row in ids.tolist()]


def bench_pass(res, reps):
    from bioreason_b200.reward_model import RewardModel
    out = {}
    for name in ("qwen3-1.7b", "qwen3-4b"):
        hf = reward_model(name)
        rm = RewardModel(copy.deepcopy(hf), "cuda")
        V = hf.config.vocab_size
        for L in (512, 2048):
            g = torch.Generator().manual_seed(L)
            ids = torch.randint(0, V - 8, (8, L), generator=g)
            lens = torch.randint(L // 2, L + 1, (8,), generator=g)
            lens[0] = L
            mask = (torch.arange(L)[None, :] < lens[:, None]).long()
            ids[mask == 0] = hf.config.pad_token_id
            ids_d, mask_d = ids.cuda(), mask.cuda()
            calls = {"ours": lambda: rm(ids_d, mask_d),
                     "hf_bf16_sdpa": lambda: hf(input_ids=ids_d, attention_mask=mask_d)}
            with torch.no_grad():
                for f in calls.values():
                    f(); f()
                t = {k: [] for k in calls}
                for _ in range(reps):
                    for k, f in calls.items():
                        t[k].append(timed_ms(f))
            tokens = int(mask.sum())
            n_params = sum(p.numel() for p in rm._dec.layers[0].__dict__.values() if torch.is_tensor(p)) * len(rm._dec.layers)
            key = f"{name}_B8_L{L}"
            out[key] = {k: round(median(v), 3) for k, v in t.items()}
            out[key]["speedup"] = round(median(t["hf_bf16_sdpa"]) / median(t["ours"]), 3)
            # 2 FLOP per weight per token in the layer GEMMs, padded tokens included (both paths run them)
            out[key]["layer_gemm_tflop"] = round(2 * n_params * 8 * L / 1e12, 3)
            out[key]["valid_tokens"] = tokens
        del hf, rm
        torch.cuda.empty_cache()
    res["pass_ms"] = out


def bench_step(res, reps, completion):
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.synth import synth_batch
    from bioreason_b200.trainer import DNALLMGRPOConfig
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer
    tc, dc = text_config("qwen3-4b"), dna_config("nt-v2-500m")
    G, C = 8, completion
    m = DNALLMModel(tc, dc, seed=1234)
    m.enable_lora(r=32, alpha=64.0, seed=3)
    with torch.no_grad():
        for p in m._lora.params[1::2]:
            p.normal_(0, 0.01)
    m.sync_adapters(rollout=False)
    b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
    P = b["input_ids"].shape[1]
    prompt = " ".join(f"w{t % N_WORDS}" for t in b["input_ids"][0].tolist()) + " "
    batch = dict(input_ids=b["input_ids"], attention_mask=b["attention_mask"], dna_tokenized=b["dna_tokenized"],
                 batch_idx_map=b["batch_idx_map"], prompts=[prompt] * G)
    res.update(step_model="qwen3-4b", rows=G, C=C, P=P, reward_model="qwen3-1.7b")

    def reward(completion_ids, **kw_):
        return (completion_ids % 7 == 0).float().sum(1)
    base = dict(num_generations=G, max_completion_length=C, per_device_train_batch_size=G, suppress_eos=True, beta=0.04,
                learning_rate=1e-6, lora_r=32, lora_alpha=64.0)
    trainers = {"callable_only": DNALLMGRPOTrainer(m, [reward], DNALLMGRPOConfig(**base), processing_class=WordTok()),
                "with_reward_model": DNALLMGRPOTrainer(m, [reward, reward_model("qwen3-1.7b", seed=5)], DNALLMGRPOConfig(**base),
                                                       processing_class=WordTok(), reward_processing_classes=[None, word_tokenizer()])}
    steps = {k: [] for k in trainers}
    for rep in range(reps + 1):                                              # rep 0: warm-up (weights, decode graph)
        for name, tr in trainers.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.training_step(batch)
            torch.cuda.synchronize()
            if rep:
                steps[name].append(time.perf_counter() - t0)
    res["training_step_s"] = {k: [round(t, 4) for t in v] for k, v in steps.items()}
    res["training_step_median_s"] = {k: round(median(v), 4) for k, v in steps.items()}
    res["step_overhead_pct"] = round(100 * (median(steps["with_reward_model"]) / median(steps["callable_only"]) - 1), 3)
    res["reward_host_s_per_step"] = round(trainers["with_reward_model"].timings["reward_host"] / (reps + 1), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--completion", type=int, default=512)
    ap.add_argument("--no-train", action="store_true", help="skip the training_step timings")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    from bioreason_b200.build import ensure_built
    ensure_built()
    res = {"card": card()}
    bench_pass(res, args.reps)
    if not args.no_train:
        bench_step(res, args.reps, args.completion)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
