"""Dense versus shared-prefix GRPO passes at config (c) (Qwen3-4B, 36 layers, random init, 1 prompt x G = 8, P = 1852, C = 512, EOS
suppressed): the reference-policy log-probs, the policy forward and the policy backward, each with its peak allocation, then one full
training_step with share_prompt_prefix off and on.  The two paths alternate in one process after a warm-up; GPU times are CUDA events.
Prints one JSON object, with the card name and power limit it was measured on.

    python scripts/shared_prefix_bench.py [--reps 3] [--out FILE]
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


def timed(fn):
    """(result, GPU ms, peak bytes allocated during the call)"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1), torch.cuda.max_memory_allocated()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--text", default="qwen3-4b")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from bioreason_b200.build import ensure_built
    ensure_built()
    from bioreason_b200 import training
    from bioreason_b200.configs import dna_config, text_config
    from bioreason_b200.models import DNALLMModel
    from bioreason_b200.synth import synth_batch
    from bioreason_b200.trainer import DNALLMGRPOConfig
    from bioreason_b200.trainer.grpo_trainer import DNALLMGRPOTrainer, _slice_mm
    tc, dc = text_config(args.text), dna_config("nt-v2-500m")
    G, C = 8, 512
    m = DNALLMModel(tc, dc, seed=1234)
    m.enable_lora(r=32, alpha=64.0, seed=3)
    with torch.no_grad():
        for p in m._lora.params[1::2]:
            p.normal_(0, 0.01)
    m.sync_adapters(rollout=False)
    b = synth_batch(tc, dc, batch=G, n_seq=2, dna_len=668, text_len=512, seed=8, same_prompt=True)
    P = b["input_ids"].shape[1]
    comp = torch.randint(0, tc.eos_token_id, (G, C), generator=torch.Generator().manual_seed(9))
    ids = torch.cat([b["input_ids"], comp], 1).cuda()
    mask = torch.ones_like(ids)
    L = ids.shape[1]
    mm = dict(dna_tokenized={k: v.cuda() for k, v in b["dna_tokenized"].items()}, batch_idx_map=b["batch_idx_map"])
    wgt = torch.randn(G, C, device="cuda")
    mr_dense = DNALLMGRPOTrainer._auto_micro_rows(m, G, L)
    mr_shared = DNALLMGRPOTrainer._auto_micro_groups(m, 1, G, P, L)
    plan = training.plan_shared_prefix(G, P, L, *[t.cuda() for t in (torch.zeros(G, dtype=torch.int32), torch.full((G,), L, dtype=torch.int32))])

    def ref_pass(gs):
        with torch.no_grad():
            return training.policy_forward(m, ids, mask, mm["dna_tokenized"], mm["batch_idx_map"], C, save=False, lora=None, group_size=gs)[0]

    def fwd_bwd(gs):
        """policy forward / backward GPU ms summed over the row chunks, and the peak of each"""
        mr = mr_shared if gs else mr_dense
        m.zero_grad_buffers()
        t_f = t_b = 0.0
        pk_f = pk_b = 0
        for lo in range(0, G, mr):
            hi = min(G, lo + mr)
            mc = _slice_mm(mm, lo, hi)
            (lp, ctx), tf, pf = timed(lambda: training.policy_forward(m, ids[lo:hi], mask[lo:hi], mc["dna_tokenized"], mc["batch_idx_map"], C,
                                                                      group_size=gs))
            _, tb, pb = timed(lambda: training.policy_backward(m, ctx, wgt[lo:hi]))
            del ctx, lp
            t_f, t_b, pk_f, pk_b = t_f + tf, t_b + tb, max(pk_f, pf), max(pk_b, pb)
        return t_f, t_b, pk_f, pk_b

    res = {"card": card(), "rows": G, "P": P, "C": C, "L": L, "layers": tc.num_hidden_layers, "r": 32,
           "Lp": plan.Lp, "Ls": plan.Ls, "tokens_dense": G * L, "tokens_shared": plan.N,
           "micro_rows": {"dense": mr_dense, "shared": mr_shared}}
    for gs in (None, G):                                                    # warm-up of both paths
        ref_pass(gs); fwd_bwd(gs)
    rec = {k: {"dense": [], "shared": []} for k in ("ref_ms", "ref_peak_GB", "fwd_ms", "fwd_peak_GB", "bwd_ms", "bwd_peak_GB")}
    for _ in range(args.reps):
        for name, gs in (("dense", None), ("shared", G)):
            _, t, pk = timed(lambda: ref_pass(gs))
            rec["ref_ms"][name].append(t); rec["ref_peak_GB"][name].append(pk / 1e9)
            tf, tb, pf, pb = fwd_bwd(gs)
            rec["fwd_ms"][name].append(tf); rec["fwd_peak_GB"][name].append(pf / 1e9)
            rec["bwd_ms"][name].append(tb); rec["bwd_peak_GB"][name].append(pb / 1e9)
    res.update(rec)
    res["median_ms"] = {k: {n: sorted(v)[len(v) // 2] for n, v in rec[k].items()} for k in ("ref_ms", "fwd_ms", "bwd_ms")}

    # one full GRPO training_step each way (rollout included), fixed token rewards, micro_rows chosen by the trainer
    def reward(completion_ids, **kw):
        return (completion_ids % 7 == 0).float().sum(1)
    batch = dict(input_ids=b["input_ids"], attention_mask=b["attention_mask"], dna_tokenized=b["dna_tokenized"], batch_idx_map=b["batch_idx_map"])
    trainers = {}
    for name, flag in (("dense", False), ("shared", True)):
        cfg = DNALLMGRPOConfig(num_generations=G, max_completion_length=C, per_device_train_batch_size=G, suppress_eos=True, beta=0.04,
                               learning_rate=1e-6, lora_r=32, lora_alpha=64.0, share_prompt_prefix=flag)
        trainers[name] = DNALLMGRPOTrainer(m, [reward], cfg)
    for tr in trainers.values():                                            # warm-up (captures the decode graph once)
        tr.training_step(batch); tr.gpu_phase_ms()
    steps = {"dense": [], "shared": []}
    phases = {}
    for _ in range(args.reps):
        for name, tr in trainers.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.training_step(batch)
            torch.cuda.synchronize()
            steps[name].append(time.perf_counter() - t0)
            phases[name] = tr.gpu_phase_ms()
    res["training_step_s"] = steps
    res["training_step_phases_ms_last"] = phases
    res["grpo_tokens_per_s_median"] = {n: G * C / sorted(v)[len(v) // 2] for n, v in steps.items()}     # bench.py's count: rows x C
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
