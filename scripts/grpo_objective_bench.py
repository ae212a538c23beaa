"""Cost of the GRPO objectives of later TRL releases (br_grpo_objective_fwd_bwd) against the default loss kernel.

  - kernel: CUDA-event time per call of br_grpo_objective_fwd_bwd (token and sequence level, dapo normaliser, delta, with the
    gradient) against br_grpo_loss_fwd_bwd, at B = 8, C = 512 and B = 32, C = 4096, mu = 2, beta = 0.04;
  - config (c) (Qwen3-4B, random init, LoRA r = 32, 1 prompt x G = 8, P = 1852, C = 512, EOS suppressed): training_step wall time
    with loss_type="dapo", importance_sampling_level="sequence" against the defaults, the two trainers alternating step by step on one
    model in one process after a warm-up step each.
Prints one JSON object with the card name and power limit it was measured on.

    python scripts/grpo_objective_bench.py [--reps 5] [--no-train] [--out FILE]
"""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:                                                  # the numbers stay usable without it
        return f"unknown ({e})"


def events_us(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


def median(v):
    return sorted(v)[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--text", default="qwen3-4b")
    ap.add_argument("--completion", type=int, default=512)
    ap.add_argument("--no-train", action="store_true", help="skip the training_step timings")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import ops
    res = {"card": card()}

    # ---- the loss kernels alone
    kern = {}
    for B, C in ((8, 512), (32, 4096)):
        g = torch.Generator(device="cuda").manual_seed(B)
        lp = -torch.rand(B, C, device="cuda", generator=g) * 4
        old = lp + torch.randn(B, C, device="cuda", generator=g) * 0.2
        ref = lp + torch.randn(B, C, device="cuda", generator=g) * 0.3
        adv = torch.randn(B, device="cuda", generator=g)
        mask = torch.ones(B, C, device="cuda", dtype=torch.int32)
        norm = torch.tensor([float(B * C)], device="cuda")
        calls = {
            "grpo_loss": lambda: ops.grpo_loss_raw(lp, old, ref, adv, mask, 0.04, 0.2, 0.2),
            "objective_token_grpo": lambda: ops.grpo_objective_raw(lp, old, ref, adv, mask, 0.04, 0.2, 0.2, norm_rows=B),
            "objective_token_dapo_delta": lambda: ops.grpo_objective_raw(lp, old, ref, adv, mask, 0.04, 0.2, 0.2, norm=norm, delta=2.0),
            "objective_sequence_dapo": lambda: ops.grpo_objective_raw(lp, old, ref, adv, mask, 0.04, 0.2, 0.2, norm=norm, sequence_level=True),
        }
        for f in calls.values():
            events_us(f, 20)
        t = {k: [] for k in calls}
        for _ in range(args.reps):
            for k, f in calls.items():
                t[k].append(events_us(f, 200))
        kern[f"B{B}_C{C}"] = {k: round(median(v), 2) for k, v in t.items()}
    res["kernel_us_per_call"] = kern

    # ---- config (c) training_step, dapo + sequence level against the defaults, alternating
    if not args.no_train:
        from bioreason_b200.configs import dna_config, text_config
        from bioreason_b200.models import DNALLMModel
        from bioreason_b200.synth import synth_batch
        from bioreason_b200.trainer import DNALLMGRPOConfig
        from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer
        tc, dc = text_config(args.text), dna_config("nt-v2-500m")
        G, C = 8, args.completion
        m = DNALLMModel(tc, dc, seed=1234)
        m.enable_lora(r=32, alpha=64.0, seed=3)
        with torch.no_grad():
            for p in m._lora.params[1::2]:
                p.normal_(0, 0.01)
        m.sync_adapters(rollout=False)
        b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
        batch = dict(input_ids=b["input_ids"], attention_mask=b["attention_mask"], dna_tokenized=b["dna_tokenized"],
                     batch_idx_map=b["batch_idx_map"])
        res.update(model=args.text, rows=G, C=C, P=b["input_ids"].shape[1])

        def reward(completion_ids, **kw_):
            return (completion_ids % 7 == 0).float().sum(1)
        base = dict(num_generations=G, max_completion_length=C, per_device_train_batch_size=G, suppress_eos=True, beta=0.04,
                    learning_rate=1e-6, lora_r=32, lora_alpha=64.0)
        trainers = {"default": DNALLMGRPOTrainer(m, [reward], DNALLMGRPOConfig(**base)),
                    "dapo_sequence": DNALLMGRPOTrainer(m, [reward], DNALLMGRPOConfig(loss_type="dapo", importance_sampling_level="sequence", **base))}
        steps = {k: [] for k in trainers}
        for rep in range(args.reps + 1):                                    # rep 0: warm-up (weights, decode graph)
            for name, tr in trainers.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tr.training_step(batch)
                torch.cuda.synchronize()
                if rep:
                    steps[name].append(time.perf_counter() - t0)
        res["training_step_s"] = {k: [round(t, 4) for t in v] for k, v in steps.items()}
        res["training_step_median_s"] = {k: round(median(v), 4) for k, v in steps.items()}
        res["step_overhead_pct"] = round(100 * (median(steps["dapo_sequence"]) / median(steps["default"]) - 1), 3)
        res["metrics_dapo_sequence"] = {k: round(v, 6) for k, v in trainers["dapo_sequence"].log_metrics().items()
                                        if k.startswith(("clip_ratio", "kl"))}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
