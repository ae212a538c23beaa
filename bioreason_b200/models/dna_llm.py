"""CUDA-native `DNALLMModel` -- same Python surface as bioreason/models/dna_llm.py:18-305, math in libbioreason_b200.

What is kept from the reference (SURVEY.md §8b): constructor kwargs, `forward(input_ids, attention_mask, dna_tokenized,
batch_idx_map, labels=None, **kw)` returning an object with `.logits` / `.loss`, `generate(...)` returning completion-only
ids, the two ValueErrors, and the attributes callers touch (`text_model`, `dna_model`, `dna_projection`, `text_config`,
`dna_config`, `dna_token_id`, `max_length_*`, `text_hidden_size`, `dna_hidden_size`).  `text_model` / `dna_model` are the
HF module trees (state_dict keys, `named_modules()` with nn.Linear leaves, `.config`) whose storage is re-pointed into
the fused kernel layout (packing.py); their own `forward` is never on the product path.

What differs by design: the encoder's unused MLM head is skipped, the per-sequence `.item()` syncs are gone (one
combined count check per call), and logits are materialised lazily -- `per_token_logps()` and `.loss` use the fused
lm_head + log-sum-exp kernel and never write [B, L, V] to HBM.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional

import torch
import torch.nn as nn

from .. import engine, ops
from ..configs import dna_config as _dna_config
from ..configs import text_config as _text_config
from ..packing import LINEARS, gu_views, pack_decoder, pack_encoder, refresh_decoder_gu

_TEXT_ALIASES = {"Qwen/Qwen3-4B": "qwen3-4b", "Qwen/Qwen3-1.7B": "qwen3-1.7b"}
_DNA_ALIASES = {"InstaDeepAI/nucleotide-transformer-v2-500m-multi-species": "nt-v2-500m"}


def _config_from_dir(path: str, kind: str):
    """config.json of a local HF checkpoint directory -> the config object the kernels are built from (no hub access)."""
    import json
    from transformers import EsmConfig, Qwen3Config
    raw = json.load(open(os.path.join(path, "config.json")))
    if kind == "text":
        cfg = Qwen3Config(**{k: v for k, v in raw.items() if k not in ("architectures", "model_type", "transformers_version", "torch_dtype", "auto_map")})
        if getattr(cfg, "dna_token_ids", None) is None:
            from ..configs import DNA_END_ID, DNA_PAD_ID, DNA_START_ID
            cfg.dna_token_ids = (DNA_START_ID, DNA_PAD_ID, DNA_END_ID)
        if cfg.pad_token_id is None:
            cfg.pad_token_id = cfg.eos_token_id if not isinstance(cfg.eos_token_id, (list, tuple)) else cfg.eos_token_id[0]
        cfg._attn_implementation = "sdpa"
        return cfg
    cfg = EsmConfig(**{k: v for k, v in raw.items() if k not in ("architectures", "model_type", "transformers_version", "torch_dtype", "auto_map")})
    cfg.gated_mlp = True                                                    # NT-v2 (SURVEY.md §8.0); plain ESM FFNs are not on this path
    cfg.add_bias_fc = bool(raw.get("add_bias_fc", False))
    if getattr(cfg, "cls_token_id", None) is None:
        cfg.cls_token_id = 3
    cfg._attn_implementation = "sdpa"
    return cfg


class LazyCausalLMOutput:
    """`.logits` ([B, L, V]) is computed on first access; `.loss` comes from the fused CE kernel."""

    def __init__(self, model, hidden, B, L, loss=None):
        self._model, self._hidden, self._B, self._L = model, hidden, B, L
        self.loss = loss
        self._logits = None

    @property
    def logits(self):
        if self._logits is None:
            W = self._model._dec
            self._logits = ops.gemm(self._hidden, W.lm_head).view(self._B, self._L, -1)
        return self._logits

    @property
    def hidden_states(self):
        return self._hidden.view(self._B, self._L, -1)


class DNALLMModel(nn.Module):
    def __init__(self, text_model_name, dna_model_name, cache_dir: Optional[str] = None, max_length_dna: int = 2048,
                 max_length_text: int = 512, text_model_finetune: bool = True, dna_model_finetune: bool = True,
                 dna_is_evo2: bool = False, dna_embedding_layer: str = None, *, seed: int = 1234, device="cuda", **kwargs):
        # **kwargs absorbs `debug=False` passed by reason.py:418 (not in the reference signature either)
        super().__init__()
        if dna_is_evo2:
            raise NotImplementedError("Evo2 (StripedHyena-2) encoder is SURVEY.md §8f 'next'; NT-v2 is the path built here")
        if not torch.cuda.is_available():
            raise RuntimeError("bioreason_b200.DNALLMModel needs a CUDA device (sm_90a); there is no CPU fallback")
        self.text_model_finetune, self.dna_model_finetune = text_model_finetune, dna_model_finetune
        self.max_length_dna, self.max_length_text = max_length_dna, max_length_text
        self.dna_is_evo2, self.dna_embedding_layer = dna_is_evo2, dna_embedding_layer
        self.warnings_issued = {}                                           # grpo_trainer.py:411 writes into it
        self._local_dirs = []
        text_model, dna_model = self._build_modules(text_model_name, dna_model_name, cache_dir, seed, self._local_dirs)
        self.text_model, self.dna_model = text_model, dna_model
        # back-reference for compat/peft.get_peft_model(model.text_model, ...) (reason.py:386): plain attribute, not a submodule
        object.__setattr__(text_model, "_b200_owner", __import__("weakref").ref(self))
        self.text_config, self.dna_config = text_model.config, dna_model.config
        self.config = self.text_config                                      # grpo_trainer.py:472 touches model.config
        self.text_tokenizer = self.dna_tokenizer = self.processor = None    # no tokenizer files offline
        self.text_hidden_size, self.dna_hidden_size = self.text_config.hidden_size, self.dna_config.hidden_size
        g = torch.Generator().manual_seed(seed + 7)
        self.dna_projection = nn.Linear(self.dna_hidden_size, self.text_hidden_size)     # dna_llm.py:97 (fp32 master)
        with torch.no_grad():
            bound = self.dna_hidden_size ** -0.5
            self.dna_projection.weight.copy_((torch.rand(self.dna_projection.weight.shape, generator=g) * 2 - 1) * bound)
            self.dna_projection.bias.copy_((torch.rand(self.dna_projection.bias.shape, generator=g) * 2 - 1) * bound)
        self.dna_projection.to(device)
        ids = getattr(self.text_config, "dna_token_ids", None)
        self.dna_token_id = ids[1] if ids else None
        self._dec = pack_decoder(self.text_model, device)
        self._enc = pack_encoder(self.dna_model, device)
        self._proj_w16 = self._proj_b16 = None
        self._lora = None
        self._proj_ref = None
        self._rollout_dec = None
        self._fp8_rollout = False
        self._proj_grad_w = torch.zeros_like(self.dna_projection.weight, dtype=torch.float32)
        self._proj_grad_b = torch.zeros_like(self.dna_projection.bias, dtype=torch.float32)
        self.sync_projection()
        for prefix, path in self._local_dirs:                               # local HF checkpoint directories (dna_llm.py:57-68)
            from .. import checkpoint
            sd = {prefix + k: v for k, v in checkpoint.read_hf_dir(path).items()}
            mapped, _ = checkpoint.normalize_keys(sd, self.state_dict().keys())
            self.load_weights(mapped)

    @property
    def text(self):
        """reason.py:89 walks `model.text.named_modules()`."""
        return self.text_model

    # ------------------------------------------------------------------ construction helpers
    @staticmethod
    def _build_modules(text_name, dna_name, cache_dir, seed, local_dirs):
        from transformers import EsmForMaskedLM, Qwen3ForCausalLM
        def resolve(name, aliases, factory, kind):
            if not isinstance(name, str):
                return name                                                  # a config object
            if os.path.isdir(name):                                          # local HF checkpoint directory: config.json + weights
                local_dirs.append(("text_model." if kind == "text" else "dna_model.", name))
                return _config_from_dir(name, kind)
            key = aliases.get(name, name)
            return factory(key)
        tcfg = resolve(text_name, _TEXT_ALIASES, _text_config, "text")
        dcfg = resolve(dna_name, _DNA_ALIASES, _dna_config, "dna")
        # seeded random init at the real shapes (no weights exist offline); built directly on the GPU in bf16
        dt = torch.get_default_dtype()
        try:
            torch.set_default_dtype(torch.bfloat16)
            with torch.device("cuda"):
                torch.manual_seed(seed)
                text = Qwen3ForCausalLM(tcfg)
                torch.manual_seed(seed + 1)
                dna = EsmForMaskedLM(dcfg)
                if getattr(dcfg, "gated_mlp", False):
                    for layer in dna.esm.encoder.layer:
                        F, d = dcfg.intermediate_size, dcfg.hidden_size
                        layer.intermediate.dense = nn.Linear(d, 2 * F, bias=getattr(dcfg, "add_bias_fc", False))
                        layer.output.dense = nn.Linear(F, d, bias=getattr(dcfg, "add_bias_fc", False))
                        nn.init.normal_(layer.intermediate.dense.weight, std=0.02)
                        nn.init.normal_(layer.output.dense.weight, std=0.02)
        finally:
            torch.set_default_dtype(dt)
        return text.eval(), dna.eval()

    @classmethod
    def from_oracle(cls, oracle_model, device="cuda"):
        """Test helper: adopt the weights of an oracle/HF-shaped model (same state_dict keys) so both sides compute
        on identical parameters."""
        tc, dc = oracle_model.text_config, oracle_model.dna_config
        self = cls(tc, dc, device=device)
        self.load_weights({k: v for k, v in oracle_model.state_dict().items()})
        return self

    def load_state_dict(self, state_dict, strict: bool = False, assign: bool = False):
        """torch's signature; accepts every checkpoint layout the reference's scripts read (reason.py:448-537, see checkpoint.py) and
        refreshes the kernel-layout copies.  Returns the usual (missing_keys, unexpected_keys) pair."""
        from .. import checkpoint
        return checkpoint.load_into(self, state_dict, strict=strict)

    def load_checkpoint(self, path):
        """A PyTorch file (raw / Lightning / DeepSpeed state dict), a peft adapter directory or a HF model directory."""
        from .. import checkpoint
        return checkpoint.load_into(self, path)

    def load_weights(self, state_dict: Dict[str, torch.Tensor]):
        """load_state_dict(strict=False) that tolerates the NT-v2 FFN layout and refreshes kernel-layout copies.
        Returns the list of this model's keys the dict did not cover."""
        own = self.state_dict()
        seen = set()
        with torch.no_grad():
            for k, v in state_dict.items():
                if k in own and own[k].shape == v.shape:
                    own[k].copy_(v.to(device=own[k].device, dtype=own[k].dtype))
                    seen.add(k)
        missing = [k for k in own if k not in seen and "inv_freq" not in k and "position_ids" not in k]
        # the encoder's interleaved gate/up copy and the projector compute copy are derived -> rebuild
        F = self.dna_config.intermediate_size
        with torch.no_grad():
            for layer, Lw in zip(self.dna_model.esm.encoder.layer, self._enc.layers):
                w = layer.intermediate.dense.weight.data
                gv, uv = gu_views(Lw.w_gu)
                gv.copy_(w[:F].view(F // 8, 8, -1)); uv.copy_(w[F:].view(F // 8, 8, -1))
        refresh_decoder_gu(self.text_model, self._dec)
        self._rollout_dec = None
        self._enc_cache = None
        if getattr(self, "_rollout", None) is not None:
            self._rollout._cached.clear()
        self.sync_projection()
        if self._lora is not None:
            self._dec.build_transposes()
            self.sync_adapters(rollout=False)
        return missing

    def sync_projection(self):
        """bf16 compute copy of the (fp32 master) projector; call after every optimizer step."""
        self._proj_w16 = self.dna_projection.weight.detach().to(torch.bfloat16).contiguous()
        self._proj_b16 = self.dna_projection.bias.detach().to(torch.bfloat16).contiguous()

    # ------------------------------------------------------------------ adapters / training state
    def enable_lora(self, r: int = 32, alpha: float = 64.0, seed: int = 0):
        """What `get_peft_model(model.text_model, LoraConfig(r=32, lora_alpha=64, target_modules=<all linears>))`
        does in reason.py:376-388, in kernel layout.  Freezes the base text model and the DNA encoder."""
        from ..lora import LoraState
        self._lora = LoraState(self.text_model, self._dec, r, alpha, seed)
        # Rollout weights built before the adapters existed alias the frozen base w_o / w_down (nothing to merge then); a later
        # merge into that object would write W + s*B*A INTO the base weights.  Drop them (and the decode graphs captured on them).
        self._rollout_dec = None
        if getattr(self, "_rollout", None) is not None:
            self._rollout._cached.clear()
        for p in self.dna_model.parameters():
            p.requires_grad_(False)                                          # reason.py:371-372
        self._proj_ref = (self._proj_w16.clone(), self._proj_b16.clone())    # the reference policy's projector (deep copy at init)
        self._dec.build_transposes()
        return self._lora

    def set_lora_dropout(self, p: float, seed: int = 0):
        """peft's lora_dropout for the training passes (reason.py:376-384): p = 0 (the default) turns it off, 0 < p < 1 turns it on
        with per-rank masks drawn from `seed`.  Needs the adapters (enable_lora / get_peft_model) first."""
        if self._lora is None:
            raise RuntimeError("set_lora_dropout needs LoRA adapters: call enable_lora first")
        self._lora.set_dropout(p, seed)

    def set_fp8_rollout(self, enabled: bool):
        """Weight-only FP8 for the rollout decode (off by default): the decode's qkv / o / gate-up / down matrices of every layer are
        stored as e4m3 with one fp32 scale per output row and streamed at half the bytes; the embedding, the lm_head, the prefill
        and every training / scoring pass stay bf16.  Rollouts then sample from the quantized policy.  Toggling drops the rollout
        weights and the decode graphs captured on them; the next rollout rebuilds them in the new format."""
        enabled = bool(enabled)
        if enabled != getattr(self, "_fp8_rollout", False):
            self._fp8_rollout = enabled
            self._rollout_dec = None
            if getattr(self, "_rollout", None) is not None:
                self._rollout._cached.clear()

    def new_lora_dropout_pass(self) -> Optional[int]:
        """Pass id shared by the row chunks of one dropout-applying pass (None while dropout is off)."""
        if self._lora is None or self._lora.dropout is None:
            return None
        return self._lora.new_dropout_pass()

    @torch.no_grad()
    def merge_and_unload_lora(self):
        """peft's `merge_and_unload()` (reason.py:443-446): W <- W + (alpha/r) B A for every adapted projection, then drop the adapters
        (the merged model becomes the new frozen base / reference policy)."""
        if self._lora is None:
            return
        s = self._lora.scale
        for layer, mods in zip(self.text_model.model.layers, self._lora.modules):
            for f in LINEARS:
                parent = getattr(layer, f.parent)
                for n in f.targets:
                    ll = mods[n]
                    w = ll.base_layer.weight
                    w.data.add_((s * (ll.lora_B["default"].weight.float() @ ll.lora_A["default"].weight.float())).to(w.dtype))
                    setattr(parent, n, ll.base_layer)
        self._lora, self._proj_ref, self._rollout_dec = None, None, None
        if getattr(self, "_rollout", None) is not None:
            self._rollout._cached.clear()
        refresh_decoder_gu(self.text_model, self._dec)                      # gate/up kernel copy + stale transposes

    def trainable_parameters(self):
        ps = list(self._lora.params) if self._lora is not None else []
        return ps + [self.dna_projection.weight, self.dna_projection.bias]

    def zero_grad_buffers(self):
        if self._lora is not None:
            self._lora.zero_grad()
        self._proj_grad_w.zero_(); self._proj_grad_b.zero_()

    def attach_grads(self):
        """Point every trainable parameter's .grad at the buffers the backward kernels accumulated into."""
        if self._lora is not None:
            self._lora.attach_grads()
        self.dna_projection.weight.grad = self._proj_grad_w
        self.dna_projection.bias.grad = self._proj_grad_b

    def sync_adapters(self, rollout: bool = True):
        """After an optimizer step: refresh the bf16 kernel-layout copies (LoRA, projector) and the merged rollout weights."""
        self.sync_projection()
        if self._lora is not None:
            self._lora.sync()
            if rollout:
                from ..lora import build_rollout_weights, build_rollout_weights_fp8
                build = build_rollout_weights_fp8 if getattr(self, "_fp8_rollout", False) else build_rollout_weights
                self._rollout_dec = build(self._dec, self._lora, out=self._rollout_dec)

    # ------------------------------------------------------------------ hot path
    def merged_embeddings(self, input_ids, dna_tokenized, batch_idx_map, *, return_proj_inputs: bool = False):
        """dna_llm.py:211-229 + 103-179: text-embedding gather, encoder, projector GEMM whose epilogue scatters rows
        straight into the <|dna_pad|> slots (SURVEY.md K2-K4)."""
        dev = self._dec.embed.device
        input_ids = input_ids.to(dev)
        B, L = input_ids.shape
        emb = ops.embed_gather(input_ids, self._dec.embed)                  # [B*L, d]
        aux = None
        if dna_tokenized is not None and batch_idx_map:
            dna_ids = dna_tokenized["input_ids"].to(dev)
            dna_mask = dna_tokenized["attention_mask"].to(dev)
            row_map, n_feat, n_slots = engine.dna_row_map(input_ids, self.dna_token_id, dna_mask, list(batch_idx_map))
            # GRPO batches repeat every prompt G times (RepeatRandomSampler): encode each distinct DNA sequence once.  dup[i] = sequence i
            # equals sequence i - k (k sequences per batch item); the flags ride on the one host sync this call makes anyway.
            n_seq = dna_ids.shape[0]
            k = n_seq // B if B and n_seq % B == 0 and list(batch_idx_map) == [i // max(1, n_seq // B) for i in range(n_seq)] else 0
            dup = torch.zeros(n_seq, dtype=torch.long, device=dev)
            if k and n_seq > k:
                dup[k:] = ((dna_ids[k:] == dna_ids[:-k]).all(dim=1) & (dna_mask[k:] == dna_mask[:-k]).all(dim=1)).long()
            host = torch.cat([torch.stack([n_feat, n_slots]), dup]).tolist()  # the one host sync (reference: n_seq + 1)
            n_feat, n_slots, dup = host[0], host[1], host[2:]
            if n_feat != n_slots:
                raise ValueError(f"DNA features and DNA tokens do not match: features {n_feat}, tokens: {n_slots}")
            enc = self._encode_unique(dna_ids, dna_mask, dup, k)
            ops.gemm(enc, self._proj_w16, bias=self._proj_b16, out=emb, row_map=row_map)
            aux = (enc, row_map)
        return (emb, aux) if return_proj_inputs else emb

    def _encode_unique(self, dna_ids, dna_mask, dup, k):
        """Encoder output [n_seq * S, d_dna] with every distinct sequence encoded once; the result of the last call is kept and reused
        while the same id tensors come back unmodified (the frozen encoder runs under no_grad in the reference too, dna_llm.py:121):
        the reference-policy pass and the policy pass of one GRPO step share one encoder run."""
        key = (dna_ids.data_ptr(), dna_ids._version, tuple(dna_ids.shape), dna_mask.data_ptr(), dna_mask._version)
        cached = getattr(self, "_enc_cache", None)
        if cached is not None and cached[0] == key:
            return cached[1]
        n_seq, S = dna_ids.shape
        src = list(range(n_seq))
        for i in range(n_seq):
            if dup[i]:
                src[i] = src[i - k]
        uniq = sorted(set(src))
        with torch.no_grad():
            if len(uniq) == n_seq:
                enc = engine.encoder_forward(self._enc, dna_ids, dna_mask)
            else:
                ut = torch.tensor(uniq, device=dna_ids.device)
                enc_u = engine.encoder_forward(self._enc, dna_ids[ut], dna_mask[ut])
                slot = {u: j for j, u in enumerate(uniq)}
                seq_slot = torch.tensor([slot[src[i]] for i in range(n_seq)], device=dna_ids.device, dtype=torch.int32)
                rows = (seq_slot[:, None] * S + torch.arange(S, device=dna_ids.device, dtype=torch.int32)[None, :]).reshape(-1).contiguous()
                enc = ops.gather_rows(enc_u, rows)
        self._enc_cache = (key, enc, dna_ids, dna_mask)                     # the tensors are held so their storage cannot be recycled
        return enc

    def process_dna_embeddings(self, dna_tokenized: Dict[str, torch.Tensor], batch_idx_map: List[int], batch_size: int) -> List[torch.Tensor]:
        """dna_llm.py:103-179 as a standalone call: encoder (no grad) -> projector -> the first `valid_length` rows of every
        sequence, concatenated per batch item.  forward()/generate() do not go through this list form (the projector GEMM
        scatters straight into the embedding buffer); it exists for callers that want the per-item DNA embeddings."""
        dev = self._dec.embed.device
        ids = dna_tokenized["input_ids"].to(dev)
        mask = dna_tokenized["attention_mask"].to(dev)
        with torch.no_grad():
            enc = engine.encoder_forward(self._enc, ids, mask)                      # [n_seq * S, d_dna]
        proj = ops.gemm(enc, self._proj_w16, bias=self._proj_b16).view(ids.shape[0], ids.shape[1], -1)
        valid = mask.sum(dim=1).tolist()                                            # reference: one .item() per sequence (:168)
        result = [[] for _ in range(batch_size)]
        for seq_idx, batch_idx in enumerate(batch_idx_map):
            result[batch_idx].append(proj[seq_idx, : valid[seq_idx]])
        return [torch.cat(r, dim=0) if r else torch.zeros((0, self.text_hidden_size), device=dev, dtype=proj.dtype) for r in result]

    def forward(self, input_ids=None, attention_mask=None, dna_tokenized=None, batch_idx_map=None, labels=None, **kwargs):
        if input_ids is None or attention_mask is None:
            raise ValueError("Either 'inputs' or 'input_ids'/'attention_mask' must be provided")
        dev = self._dec.embed.device
        B, L = input_ids.shape
        attention_mask = attention_mask.to(dev)
        emb = self.merged_embeddings(input_ids, dna_tokenized, batch_idx_map)
        ks, ke = engine.mask_window(attention_mask)
        pos = engine.forward_positions(B, L, dev)                           # no position_ids -> arange (SURVEY.md §3.1)
        hidden = engine.decoder_forward(self._dec, emb, B, L, pos, ks, ke, lora=self._lora.w if self._lora is not None else None)
        loss = None
        if labels is not None:
            loss = self._ce_loss(hidden, labels.to(dev), B, L)
        return LazyCausalLMOutput(self, hidden, B, L, loss)

    def _ce_loss(self, hidden, labels, B, L):
        """HF ForCausalLMLoss (loss/loss_utils.py:28-67): shift, ignore -100, mean -- on the fused lm_head kernel."""
        tgt = torch.full((B, L), -1, device=labels.device, dtype=torch.int32)
        tgt[:, :-1] = torch.where(labels[:, 1:] == -100, -1, labels[:, 1:]).to(torch.int32)
        logp, _ = ops.lmhead_logprob(hidden, self._dec.lm_head, tgt.reshape(-1))
        n = (tgt >= 0).sum().clamp(min=1)
        return -(logp.sum() / n)

    def sft_step(self, input_ids, attention_mask, dna_tokenized=None, batch_idx_map=None, labels=None, backward: bool = True):
        """SFT loss (+ hand-written backward into the LoRA / projector gradient buffers); see training.sft_step."""
        from .. import training
        return training.sft_step(self, input_ids, attention_mask, dna_tokenized, batch_idx_map, labels, backward=backward)

    def per_token_logps(self, input_ids, attention_mask, dna_tokenized=None, batch_idx_map=None, keep_last: Optional[int] = None):
        """Fused equivalent of `_get_per_token_logps` (grpo_trainer.py:510-520): [B, L-1] (or the last `keep_last`
        columns, i.e. the `[:, P-1:]` slice the trainer takes) log-probs of the realised next tokens; no [B, L, V]."""
        out = self.forward(input_ids, attention_mask, dna_tokenized, batch_idx_map)
        return self.logps_from_hidden(out._hidden, input_ids, keep_last)

    @torch.no_grad()
    def generate(self, input_ids=None, attention_mask=None, dna_tokenized=None, batch_idx_map=None, **generation_kwargs):
        """dna_llm.py:246-305: completion-only ids.  Accepts loose kwargs (max_new_tokens, temperature, top_p, top_k,
        do_sample; train_dna_qwen.py:279-289; repetition_penalty, min_p, min_new_tokens / min_length, num_return_sequences) and
        `generation_config=` (grpo_trainer.py:581-584); loose kwargs win.  A non-default value of any other HF generation argument that
        could change the ids or the return type raises NotImplementedError.  Extra: `uniforms=` [max_new_tokens, B * num_return_sequences]
        for replayable sampling; `return_logprobs=True` returns (ids, logps) (and stats last with `return_stats`),
        logps [B, len] fp32 = each sampled token's log-prob under the rollout's raw logits (T = 1, full vocabulary), 0 after EOS."""
        if input_ids is None or attention_mask is None:
            raise ValueError("Either 'inputs' or 'input_ids'/'attention_mask' must be provided")
        from ..generation import RolloutEngine, SamplingParams, expand_return_sequences
        if getattr(self, "_rollout", None) is None:
            self._rollout = RolloutEngine(self)
        uniforms = generation_kwargs.pop("uniforms", None)
        use_graph = generation_kwargs.pop("use_graph", True)
        return_stats = generation_kwargs.pop("return_stats", False)
        return_logprobs = generation_kwargs.pop("return_logprobs", False)
        params = SamplingParams.from_hf_kwargs(self.text_config, generation_kwargs, prompt_width=input_ids.shape[1])
        # num_return_sequences: n consecutive copies of each row (HF's expansion); the engine's group detection prefills each prompt once
        input_ids, attention_mask, dna_tokenized, batch_idx_map = expand_return_sequences(input_ids, attention_mask, dna_tokenized,
                                                                                          batch_idx_map, params.num_return_sequences)
        return self._rollout.generate(input_ids, attention_mask, dna_tokenized, batch_idx_map, params=params, uniforms=uniforms,
                                      use_graph=use_graph, return_stats=return_stats, return_logprobs=return_logprobs)

    def logps_from_hidden(self, hidden, input_ids, keep_last=None):
        dev = hidden.device
        B, L = input_ids.shape
        n = L - 1 if keep_last is None else keep_last
        cols = torch.arange(L - 1 - n, L - 1, device=dev)
        rows = (torch.arange(B, device=dev)[:, None] * L + cols[None, :]).reshape(-1).to(torch.int32)
        h_sel = ops.gather_rows(hidden, rows)
        tgt = input_ids.to(dev)[:, L - n:].reshape(-1)
        logp, _ = ops.lmhead_logprob(h_sel, self._dec.lm_head, tgt)
        return logp.view(B, n)
