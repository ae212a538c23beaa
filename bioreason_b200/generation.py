"""Rollout engine: prefix-shared prefill + CUDA-graph decode loop on the paged-KV kernels.

Replaces `DNALLMModel.generate` -> `text_model.generate(inputs_embeds=..., use_cache=True, **kw)` (dna_llm.py:246-305; HF
generation/utils.py:2760-2800).  Semantics kept: completion-only ids; position_ids = cumsum(mask)-1 (pads excluded);
processor order repetition penalty -> min new tokens -> temperature -> top-k -> top-p -> min-p (the
penalty set holds the generated tokens only, as with inputs_embeds); finished rows emit pad; output trimmed to the longest unfinished row.
Redundancy removed (SURVEY.md §3.3): identical consecutive prompts (the G samples of a GRPO group) are encoded and
prefilled once and share their prompt KV pages.
"""
from __future__ import annotations

import gc
import math
from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional

import torch

from . import engine, ops
from .packing import DecoderW

PAGE = 64


# HF generate() arguments that cannot change the ids or the return type: accepted and ignored.  Every other GenerationConfig field that
# SamplingParams does not build is refused when it differs from HF's neutral value (_unbuilt_generation_args).
_NO_EFFECT_ARGS = frozenset({
    "use_cache", "cache_implementation", "cache_config", "compile_config", "disable_compile", "prefill_chunk_size", "low_memory",
    "continuous_batching_config", "bos_token_id", "decoder_start_token_id", "is_assistant", "transformers_version", "_from_model_config",
    "_commit_hash", "early_stopping", "length_penalty",          # beam search only (num_beams > 1 is refused)
    "output_attentions", "output_hidden_states",                 # only with return_dict_in_generate (refused)
    "num_assistant_tokens", "num_assistant_tokens_schedule", "assistant_confidence_threshold", "assistant_lookbehind",
    "target_lookbehind", "assistant_early_exit",                 # only with an assistant model (refused)
    "synced_gpus",
})
_BUILT_ARGS = frozenset({"max_new_tokens", "do_sample", "temperature", "top_k", "top_p", "eos_token_id", "pad_token_id",
                         "repetition_penalty", "min_p", "min_new_tokens", "min_length", "max_length", "num_return_sequences"})
# generate() arguments that are not GenerationConfig fields; refused unless None / empty
_CALL_ARGS = ("logits_processor", "stopping_criteria", "prefix_allowed_tokens_fn", "assistant_model", "streamer", "negative_prompt_ids",
              "negative_prompt_attention_mask", "custom_generate", "assistant_tokenizer", "tokenizer")


def _unbuilt_generation_args(kwargs, gc):
    """Names of the HF generation arguments set to a non-neutral value that the rollout does not implement (sorted).  Neutral = HF's
    default (GenerationConfig._get_default_generation_params(), else None), so a bare GenerationConfig passes."""
    from transformers import GenerationConfig
    neutral = GenerationConfig._get_default_generation_params()
    fields = set(GenerationConfig().to_dict()) | set(neutral)
    bad = set()
    for name in fields - _BUILT_ARGS - _NO_EFFECT_ARGS:
        for src in (kwargs, vars(gc) if gc is not None else {}):
            v = src.get(name, None)
            if v is not None and v != neutral.get(name, None):
                bad.add(name)
    for name in _CALL_ARGS:
        v = kwargs.get(name, None)
        if v is not None and not (isinstance(v, (list, tuple)) and len(v) == 0):
            bad.add(name)
    return sorted(bad)


# sampled rollouts with top_k above this (the top-k samplers' kept-set cap), or top_k = 0, use ops.sample_next_full
FULL_VOCAB_TOP_K = 1024


@dataclass
class SamplingParams:
    max_new_tokens: int = 20
    do_sample: bool = False
    temperature: float = 1.0
    top_k: int = 50
    top_p: float = 1.0
    eos_token_id: Optional[int] = None
    pad_token_id: Optional[int] = None
    # HF logits processors, in HF's order: repetition penalty -> min new tokens (EOS blocked while fewer generated) -> (sampling only)
    # temperature -> top-k -> top-p -> min-p
    repetition_penalty: float = 1.0
    min_p: float = 0.0
    min_new_tokens: int = 0
    num_return_sequences: int = 1       # DNALLMModel.generate repeats each row this many times before the rollout

    @classmethod
    def from_hf_kwargs(cls, model_cfg, kwargs, prompt_width: Optional[int] = None):
        """prompt_width: the padded prompt width P (HF's inputs_embeds width), which lowers min_length / max_length to new-token counts."""
        gc = kwargs.get("generation_config", None)
        bad = _unbuilt_generation_args(kwargs, gc)
        if bad:
            raise NotImplementedError(f"generate(): {', '.join(bad)} not supported by the rollout (only max_new_tokens, do_sample, temperature, "
                                      "top_k, top_p, min_p, repetition_penalty, min_new_tokens / min_length, num_return_sequences, "
                                      "eos_token_id and pad_token_id are implemented)")
        def pick(name, default):
            if name in kwargs and kwargs[name] is not None:
                return kwargs[name]
            if gc is not None and getattr(gc, name, None) is not None:
                return getattr(gc, name)
            return default
        eos = pick("eos_token_id", getattr(model_cfg, "eos_token_id", None))
        if isinstance(eos, (list, tuple)):
            uniq = sorted(set(int(e) for e in eos))
            if len(uniq) > 1:
                # HF stops a row on ANY of the ids; the sampler kernel tracks one.  Refuse instead of silently keeping the first.
                raise NotImplementedError(f"generate(): {len(uniq)} distinct eos_token_id values {uniq}; the decode kernels stop on a single id "
                                          "(the reference trainer masks on processing_class.eos_token_id, grpo_trainer.py:605) -- pass that one")
            eos = uniq[0] if uniq else None
        pad = pick("pad_token_id", getattr(model_cfg, "pad_token_id", None))
        if pad is None:
            pad = eos if eos is not None else 0
        max_new = pick("max_new_tokens", None)
        if max_new is None and pick("max_length", None) is not None:
            # HF then generates max_length - P tokens (inputs_embeds); not built
            raise NotImplementedError("generate(): max_length without max_new_tokens is not supported by the rollout; pass max_new_tokens")
        theta = float(pick("repetition_penalty", 1.0))
        if not theta > 0:
            raise ValueError(f"generate(): repetition_penalty must be a strictly positive float, got {theta}")
        min_p = float(pick("min_p", 0.0))
        if not 0.0 <= min_p <= 1.0:
            raise ValueError(f"generate(): min_p must be in [0, 1], got {min_p}")
        # HF _prepare_generated_length: min_new_tokens wins; else min_length lowered by the inputs_embeds width (the processors' input_ids
        # hold only generated tokens)
        m = pick("min_new_tokens", None)
        if m is None:
            ml = int(pick("min_length", 0))
            if ml < 0:
                raise ValueError(f"generate(): min_length must be >= 0, got {ml}")
            if ml > 0 and prompt_width is None:
                raise ValueError("generate(): min_length needs the prompt width")
            m = max(ml - int(prompt_width or 0), 0)
        m = int(m)
        if m < 0:
            raise ValueError(f"generate(): min_new_tokens must be >= 0, got {m}")
        n = int(pick("num_return_sequences", 1))
        if n < 1:
            raise ValueError(f"generate(): num_return_sequences must be >= 1, got {n}")
        do_sample = bool(pick("do_sample", False))
        if n > 1 and not do_sample:
            raise ValueError(f"generate(): greedy decoding does not support num_return_sequences = {n} (as in HF); pass do_sample=True")
        top_k = int(pick("top_k", 50) or 0)
        if top_k < 0:
            raise ValueError(f"generate(): top_k must be >= 0 (0: top-k off), got {top_k}")
        return cls(max_new_tokens=int(max_new if max_new is not None else 20), do_sample=do_sample,
                   temperature=float(pick("temperature", 1.0)), top_k=top_k, top_p=float(pick("top_p", 1.0)),
                   eos_token_id=eos, pad_token_id=pad, repetition_penalty=theta, min_p=min_p, min_new_tokens=m, num_return_sequences=n)


def expand_return_sequences(input_ids, attention_mask, dna_tokenized, batch_idx_map, n: int):
    """HF num_return_sequences: each row repeated n times in place (row b -> rows b n .. b n + n - 1), its DNA sequences with it.
    Returns (input_ids, attention_mask, dna_tokenized, batch_idx_map); the DNA stays ordered by the new row index."""
    if n == 1:
        return input_ids, attention_mask, dna_tokenized, batch_idx_map
    input_ids = input_ids.repeat_interleave(n, dim=0)
    attention_mask = attention_mask.repeat_interleave(n, dim=0)
    if dna_tokenized is not None and batch_idx_map:
        order, new_map = [], []
        for b in sorted(set(batch_idx_map)):
            mine = [i for i, x in enumerate(batch_idx_map) if x == b]
            for c in range(n):
                order += mine
                new_map += [b * n + c] * len(mine)
        idx = torch.tensor(order, dtype=torch.long)
        n_seq = len(batch_idx_map)
        dna_tokenized = {k: (v[idx.to(v.device)] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == n_seq else v)
                         for k, v in dna_tokenized.items()}
        batch_idx_map = new_map
    return input_ids, attention_mask, dna_tokenized, batch_idx_map


def detect_group_size(input_ids: torch.Tensor, dna_tokenized, batch_idx_map) -> torch.Tensor:
    """eq[i] = row i is identical to row i-1 (text ids and its DNA sequences) -- device tensor, no sync."""
    B = input_ids.shape[0]
    eq = torch.zeros(B, dtype=torch.bool, device=input_ids.device)
    if B > 1:
        eq[1:] = (input_ids[1:] == input_ids[:-1]).all(dim=1)
        if dna_tokenized is not None and batch_idx_map:
            counts = [0] * B
            for b in batch_idx_map:
                counts[b] += 1
            if len(set(counts)) == 1 and list(batch_idx_map) == sorted(batch_idx_map):
                d = dna_tokenized["input_ids"].to(input_ids.device).view(B, -1)
                eq[1:] &= (d[1:] == d[:-1]).all(dim=1)
            else:
                eq[:] = False
    return eq


def group_size_from_flags(eq: List[bool]) -> int:
    B = len(eq)
    for G in range(B, 0, -1):
        if B % G == 0 and all(eq[i] for i in range(B) if i % G != 0):
            return G
    return 1


def plan_pages(plen: List[int], G: int, C: int):
    """KV page plan of a rollout (host side, pure).  plen[u] = prompt length of unique prompt u; every prompt is sampled G times
    for C new tokens.  Full prompt pages (the first n_shared of every group; one count for all groups) are shared by the G rows
    of a group; the partially filled tail page and the pages of generated tokens are private per row.
    Returns dict(n_shared, max_pages, n_pages, table [U*G][max_pages] (lists), prefill_pages [U] (pages holding the prompt,
    i.e. row 0 of the group), tail_copies [(src_page, dst_page)] to replicate row 0's partially shared tail pages)."""
    U = len(plen)
    n_full = [l // PAGE for l in plen]
    n_shared = min(n_full) if G > 1 else 0
    priv = [math.ceil((l - n_shared * PAGE + C) / PAGE) for l in plen]
    max_pages = n_shared + max(priv)
    nxt = 0
    table = [[0] * max_pages for _ in range(U * G)]
    prefill_pages, tail_copies = [], []
    for u in range(U):
        shared = list(range(nxt, nxt + n_shared)); nxt += n_shared
        for g in range(G):
            r = u * G + g
            mine = list(range(nxt, nxt + priv[u])); nxt += priv[u]
            table[r][:n_shared] = shared
            table[r][n_shared:n_shared + priv[u]] = mine
        n_prompt_pages = math.ceil(plen[u] / PAGE)
        prefill_pages.append(table[u * G][:n_prompt_pages])
        for j in range(n_shared, n_prompt_pages):
            for g in range(1, G):
                tail_copies.append((table[u * G][j], table[u * G + g][j]))
    return dict(n_shared=n_shared, max_pages=max_pages, n_pages=nxt, table=table, prefill_pages=prefill_pages, tail_copies=tail_copies)


DECODE_ITEMS_PER_SM = 3                 # CTAs of the fused attention an SM can hold (74 KB each)


def decode_splits(R: int, G: int, Hkv: int, n_shared: int, n_sms: int):
    """(splits_shared, splits_private) of the fused decode attention (host side, pure).  Two KV tiles per work item where the
    co-residency cap allows it: both are fetched before the dependency wait, so the tile loop never waits on DRAM.  The in-kernel
    merge needs every work item co-resident, so the splits are halved until (R / G) Hkv SS + R Hkv SP <= 3 n_sms."""
    splits_shared = min(16, max(8, (n_shared + 1) // 2), n_shared) if n_shared > 0 else 0
    splits_private = 3 if n_shared > 0 else 8
    cap = DECODE_ITEMS_PER_SM * n_sms
    n_items = lambda ss, sp: (R // G) * Hkv * ss + R * Hkv * sp
    while n_items(splits_shared, splits_private) > cap and (splits_shared > 1 or splits_private > 1):
        if splits_private > 1 and (splits_private >= splits_shared or splits_shared <= 1):
            splits_private //= 2
        else:
            splits_shared = max(1, splits_shared // 2)
    return splits_shared, splits_private


class RolloutEngine:
    """Owns the KV page pool, decode scratch and the captured decode-step graph for one model."""

    def __init__(self, model):
        self.model = model
        self._graph = None
        self._graph_key = None
        self._weights = None            # DecoderW used for the rollout (base, or base+LoRA merged)
        self._cached = {}               # rollout shape key -> static buffers + captured decode graph (reused across steps)

    # ------------------------------------------------------------------
    def rollout_weights(self) -> DecoderW:
        """Merged (base + LoRA) weights with the RMSNorm gains folded in -- decode only; the prefill runs the regular
        forward (base weights + LoRA second K segment).  With the model's FP8 rollout on, the layer matrices are e4m3 (ops.Fp8Weight)."""
        m = self.model
        if getattr(m, "_rollout_dec", None) is None:
            from .lora import build_rollout_weights, build_rollout_weights_fp8
            build = build_rollout_weights_fp8 if getattr(m, "_fp8_rollout", False) else build_rollout_weights
            m._rollout_dec = build(m._dec, m._lora)
        return m._rollout_dec

    @torch.no_grad()
    def generate(self, input_ids, attention_mask, dna_tokenized=None, batch_idx_map=None, *, params: SamplingParams,
                 uniforms: Optional[torch.Tensor] = None, use_graph: bool = True, return_stats: bool = False,
                 return_logprobs: bool = False):
        """Completion ids [B, <= C]; return_logprobs: also the fp32 log-prob of each sampled token under the decode's own raw logits
        (T = 1, full vocabulary; 0 after a row's EOS), trimmed like the ids -- the behaviour log-probs of the rollout."""
        m = self.model
        W = m._dec                                                          # prefill weights
        Wd = self.rollout_weights()                                         # decode weights (merged + folded)
        cfg = W.cfg
        dev = W.embed.device
        Hq, Hkv, D, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim, cfg.hidden_size
        theta = cfg.rope_parameters["rope_theta"] if hasattr(cfg, "rope_parameters") else cfg.rope_theta
        eps = cfg.rms_norm_eps
        input_ids = input_ids.to(dev)
        attention_mask = attention_mask.to(dev)
        B, P = input_ids.shape
        C = params.max_new_tokens

        # ---- one host sync: grouping flags + prompt lengths + the layout check (left-padded rows, one contiguous run of ones ending at
        #      the last column: what `padding_side="left"` produces, grpo_trainer.py:556-565; KV placement and the first-token logits
        #      below assume it, so anything else is refused instead of generating from a pad position)
        eq = detect_group_size(input_ids, dna_tokenized, batch_idx_map)
        lens = attention_mask.sum(dim=1)
        m01 = attention_mask != 0
        layout_ok = (m01[:, -1].all() & (m01[:, 1:] >= m01[:, :-1]).all()).long().reshape(1) if P > 1 else m01[:, -1].all().long().reshape(1)
        host = torch.cat([eq.long(), lens, layout_ok]).tolist()
        if not host[2 * B]:
            raise ValueError("generate(): attention_mask must be left-padded (each row: zeros, then ones up to the last column)")
        G = group_size_from_flags([bool(x) for x in host[:B]])
        U = B // G
        plen = [int(x) for x in host[B:2 * B]][::G]                      # prompt length of each unique row

        # ---- encode + prefill the unique prompts only
        uid = torch.arange(0, B, G, device=dev)
        u_ids, u_mask = input_ids[uid], attention_mask[uid]
        if dna_tokenized is not None and batch_idx_map:
            keep = [i for i, b in enumerate(batch_idx_map) if b % G == 0]
            kt = torch.tensor(keep, device=dev)
            u_dna = {k: v.to(dev)[kt] for k, v in dna_tokenized.items() if k in ("input_ids", "attention_mask")}
            u_map = [batch_idx_map[i] // G for i in keep]
        else:
            u_dna, u_map = None, []
        emb = m.merged_embeddings(u_ids, u_dna, u_map)
        ks, ke = engine.mask_window(u_mask)
        pos = engine.generate_positions(u_mask)

        # ---- page plan: full prompt pages are shared by the group, the tail page + generated tokens are private
        plan = plan_pages(plen, G, C)
        n_shared, max_pages, n_pages = plan["n_shared"], plan["max_pages"], plan["n_pages"]
        table = torch.tensor(plan["table"], dtype=torch.int32)
        prefill_pages = [torch.tensor(p, dtype=torch.int32) for p in plan["prefill_pages"]]
        nl = len(W.layers)
        # Static buffers + the captured decode graph are cached per rollout shape: a training run replays the same graph every
        # step (no per-step capture, no graph-pool / allocator churn -- that churn showed up as multi-second host stalls).
        # the logits processors are baked into the captured sampler launch: they belong to the key
        rep_pen = params.repetition_penalty
        min_p = params.min_p if params.do_sample else 0.0                   # HF applies min-p only when sampling
        min_new = params.min_new_tokens
        # top_k = 0 (off) or above the 1024-value cap of the top-k samplers: the full-vocabulary sampler
        full_vocab = params.do_sample and (params.top_k == 0 or params.top_k > FULL_VOCAB_TOP_K)
        key = (B, G, tuple(plen), C, n_shared, max_pages, n_pages, params.do_sample, params.temperature, params.top_k, params.top_p,
               params.eos_token_id, params.pad_token_id, id(Wd), bool(use_graph), bool(return_logprobs), rep_pen, min_p, min_new)
        St = self._cached.get(key)
        hit = St is not None
        if not hit:
            if len(self._cached) >= 4:
                self._cached.clear()
            St = SimpleNamespace()
            St.table = table.to(dev)
            # zero-filled once: the unwritten slots of a partially filled page are multiplied by exact-zero probabilities in the P V
            # product, which is only harmless if they hold finite numbers (recycled allocator memory may hold NaN bit patterns)
            St.kc = torch.zeros(nl, n_pages, Hkv, PAGE, D, device=dev, dtype=torch.bfloat16)
            St.vc = torch.zeros_like(St.kc)
            St.pp_dev = [p.to(dev) for p in prefill_pages]
        table, kc, vc, pp_dev = St.table, St.kc, St.vc, St.pp_dev

        def kv_sink(li, qkv):
            for u in range(U):
                first = u * P + (P - plen[u])                             # first real token of the left-padded row
                ops.kv_write_pages(qkv[first:], plen[u], Hq, Hkv, D, pp_dev[u], kc[li], vc[li])

        hidden = engine.decoder_forward(W, emb, U, P, pos, ks, ke, kv_sink=kv_sink, lora=m._lora.w if m._lora is not None else None)
        # replicate each group's partially filled tail page to the other G-1 rows
        if plan["tail_copies"]:
            s_t = torch.tensor([a for a, _ in plan["tail_copies"]], device=dev)
            d_t = torch.tensor([b for _, b in plan["tail_copies"]], device=dev)
            kc[:, d_t] = kc[:, s_t]; vc[:, d_t] = vc[:, s_t]

        # ---- decode state
        R = B
        eos = params.eos_token_id if params.eos_token_id is not None else -1
        pad_fill = params.pad_token_id if params.pad_token_id is not None else 0
        if params.do_sample:
            if uniforms is None:
                uniforms = torch.rand(C, R, device=dev, dtype=torch.float32)
            uniforms = uniforms.to(dev).float().contiguous()
            assert uniforms.shape == (C, R)
        cur0 = torch.tensor([plen[r // G] for r in range(R)], device=dev, dtype=torch.int32)
        if not hit:
            St.tokens = torch.full((R, C), pad_fill, device=dev, dtype=torch.int64)
            St.logp = torch.zeros(R, C, device=dev, dtype=torch.float32) if return_logprobs else None
            St.next_ids = torch.zeros(R, device=dev, dtype=torch.int64)
            St.finished = torch.zeros(R, device=dev, dtype=torch.int32)
            St.step = torch.zeros(1, device=dev, dtype=torch.int32)
            St.cur_len = cur0.clone()
            St.uniforms = uniforms.clone() if params.do_sample else None
            St.scratch = ops.skinny_scratch(max(cfg.vocab_size, 2 * cfg.intermediate_size), dev)
            splits_shared, splits_private = decode_splits(R, G, Hkv, n_shared, torch.cuda.get_device_properties(dev).multi_processor_count)
            if G * (Hq // Hkv) > 32:
                raise NotImplementedError("fused decode attention handles G * Hq/Hkv <= 32 query vectors per kv head")
            St.splits = (splits_shared, splits_private)
            St.ws = ops.decode_fused_workspace(R, Hq, Hkv, D, splits_shared + splits_private, dev)
            St.attn_out = torch.empty(R, Hq * D, device=dev, dtype=torch.bfloat16)
            St.rope = ops.rope_table(max(plen) + C + 1, D, theta, dev)
            St.h = torch.empty(R, d, device=dev, dtype=torch.bfloat16)
            n_part_ = ((d + 127) // 128) * 4                                    # partial sum-of-squares rows a d-wide GEMM emits
            St.ssq_a = torch.zeros(n_part_, 32, device=dev, dtype=torch.float32)    # sum x^2 of the residual stream entering attention
            St.ssq_b = torch.zeros(n_part_, 32, device=dev, dtype=torch.float32)    # ... entering the MLP (see br_skinny_gemm)
            St.ssq_e = torch.zeros(1, 32, device=dev, dtype=torch.float32)          # ... of the embedding row (first layer)
            St.samp_ws = (ops.sample_full_workspace(R, cfg.vocab_size, dev) if full_vocab
                          else ops.sample_workspace(R, cfg.vocab_size, dev, logp=return_logprobs))
            # emitted-token bitmap of the repetition penalty (HF with inputs_embeds: only generated tokens count, not the prompt)
            St.presence = ops.presence_bitmap(R, cfg.vocab_size, dev) if rep_pen != 1.0 else None
            St.graph = None
        else:
            St.tokens.fill_(pad_fill); St.finished.zero_(); St.step.zero_(); St.cur_len.copy_(cur0)
            if return_logprobs:
                St.logp.zero_()
            if params.do_sample:
                St.uniforms.copy_(uniforms)
            if St.presence is not None:
                St.presence.zero_()                                         # outside the graph, before the first token
        tokens, next_ids, finished, step, cur_len = St.tokens, St.next_ids, St.finished, St.step, St.cur_len
        samp_kw = dict(logp=St.logp) if return_logprobs else {}
        if rep_pen != 1.0 or min_p > 0.0 or min_new > 0:
            samp_kw.update(repetition_penalty=rep_pen, min_p=min_p, min_new_tokens=min_new, presence=St.presence)
        uniforms = St.uniforms
        scratch, ws, attn_out, rope, h = St.scratch, St.ws, St.attn_out, St.rope, St.h
        ssq_a, ssq_b, ssq_e, samp_ws = St.ssq_a, St.ssq_b, St.ssq_e, St.samp_ws
        splits_shared, splits_private = St.splits
        n_part = ((d + 127) // 128) * 4

        def sample(logits):
            if full_vocab:
                ops.sample_next_full(logits, workspace=samp_ws, temperature=params.temperature, top_k=params.top_k, top_p=params.top_p,
                                     uniforms=uniforms, step=step, max_steps=C, eos_id=eos,
                                     pad_id=params.pad_token_id if params.pad_token_id is not None else 0, finished=finished, tokens=tokens,
                                     next_ids=next_ids, **samp_kw)
                return
            ops.sample_next(logits, workspace=samp_ws, temperature=params.temperature, top_k=params.top_k, top_p=params.top_p, do_sample=params.do_sample,
                            uniforms=uniforms if params.do_sample else None, step=step, max_steps=C, eos_id=eos,
                            pad_id=params.pad_token_id if params.pad_token_id is not None else 0, finished=finished, tokens=tokens,
                            next_ids=next_ids, **samp_kw)

        # ---- first token from the prefill's last position (row u replicated G times)
        last_rows = torch.tensor([u * P + P - 1 for u in range(U) for _ in range(G)], device=dev, dtype=torch.int32)
        h_last = ops.gather_rows(hidden, last_rows)
        logits = ops.skinny_gemm(h_last, W.lm_head, scratch, mode=3)             # prefill output is already final-normed
        sample(logits)
        step += 1                                                         # cur_len stays: the first generated token sits at index plen

        F = cfg.intermediate_size
        if not hit:
            St.b_qkv = torch.empty(R, (Hq + 2 * Hkv) * D, device=dev, dtype=torch.bfloat16)
            St.b_x2 = torch.empty(R, d, device=dev, dtype=torch.bfloat16)
            St.b_act = torch.empty(R, F, device=dev, dtype=torch.bfloat16)
            St.b_logits = torch.empty(R, cfg.vocab_size, device=dev, dtype=torch.float32)
        b_qkv, b_x2, b_act, b_logits = St.b_qkv, St.b_x2, St.b_act, St.b_logits

        def decode_step():
            # 5 launches per layer: qkv GEMM (folded ln1), fused attention, o_proj (+res, sum x^2), gate/up GEMM (folded ln2, SwiGLU),
            # down_proj (+res, sum x^2); RMSNorm never launches in the decode loop.
            ops.embed_gather_sumsq(next_ids, Wd.embed, h, ssq_e)
            for li, Lw in enumerate(Wd.layers):
                ops.skinny_gemm(h, Lw.w_qkv, scratch, out=b_qkv, sumsq_in=ssq_e if li == 0 else ssq_a, sumsq_in_n=1 if li == 0 else n_part, eps=eps)
                ops.decode_attn_fused(b_qkv, Lw.q_norm, Lw.k_norm, kc[li], vc[li], table, cur_len, G, Hq, Hkv, D, n_shared, splits_shared,
                                      splits_private, theta, eps, ws, attn_out, rope=rope)
                ops.skinny_gemm(attn_out, Lw.w_o, scratch, mode=1, residual=h, out=b_x2, sumsq_out=ssq_b)
                ops.skinny_gemm(b_x2, Lw.w_gu, scratch, mode=2, out=b_act, sumsq_in=ssq_b, sumsq_in_n=n_part, eps=eps)
                ops.skinny_gemm(b_act, Lw.w_down, scratch, mode=1, residual=b_x2, out=h, sumsq_out=ssq_a)
            ops.skinny_gemm(h, Wd.lm_head, scratch, mode=3, out=b_logits, sumsq_in=ssq_a, sumsq_in_n=n_part, eps=eps)
            sample(b_logits)
            ops.decode_advance(step, cur_len)

        n_steps = C - 1
        if not hit:
            St.decode_step = decode_step
            St.per_replay = 0
            if use_graph and n_steps > 2:
                # warm up once on a side stream (allocator + lazy func attributes), then capture one decode step
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                live = tuple(t for t in (tokens, next_ids, finished, step, cur_len, St.presence) if t is not None)
                state = [t.clone() for t in live]
                with torch.cuda.stream(s):
                    decode_step()
                torch.cuda.current_stream().wait_stream(s)
                for t, v in zip(live, state):
                    t.copy_(v)                                                # the warm-up step is replayed for real below
                St.graph = torch.cuda.CUDAGraph()
                n0 = ops.LAUNCHES[0]
                # A dropped model and its engine reference each other, so their captured graphs live until the cyclic collector
                # runs, and destroying a graph while a stream captures invalidates the capture: collect now, not inside the capture.
                gc_was_enabled = gc.isenabled()
                gc.collect()
                gc.disable()
                try:
                    with torch.cuda.graph(St.graph):
                        decode_step()
                finally:
                    if gc_was_enabled:
                        gc.enable()
                St.per_replay = ops.LAUNCHES[0] - n0
                ops.LAUNCHES[0] = n0
                for t, v in zip(live, state):
                    t.copy_(v)
            self._cached[key] = St
        graph, per_replay, decode_step = St.graph, St.per_replay, St.decode_step
        done_steps = 0
        check_every = 16
        while done_steps < n_steps:
            chunk = min(check_every, n_steps - done_steps) if eos >= 0 else n_steps - done_steps
            for _ in range(chunk):
                if graph is not None:
                    graph.replay()
                    ops.LAUNCHES[0] += per_replay
                else:
                    decode_step()
            done_steps += chunk
            if eos >= 0 and done_steps < n_steps and bool(finished.min().item() == 1):
                break
        out = tokens.clone()                                                 # the static buffer is reused by the next rollout
        if eos >= 0:
            # HF stops as soon as every row has finished: trim to the longest row (eos position inclusive)
            is_eos = out == eos
            first = torch.where(is_eos.any(1), is_eos.int().argmax(1) + 1, torch.full((R,), min(done_steps + 1, C), device=dev))
            out = out[:, : int(first.max().item())]
        res = (out, St.logp[:, : out.shape[1]].clone()) if return_logprobs else (out,)
        if return_stats:
            res += (dict(G=G, unique_prompts=U, n_shared_pages=n_shared, pages=n_pages, graph=graph is not None),)
        return res if len(res) > 1 else out
