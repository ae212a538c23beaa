"""NumPy restatement of the LoRA-dropout mask (test infrastructure; the rule is next to br_lora_dropout in include/bioreason_b200.h)
and a helper that makes the fp32 oracle's LoRA linears carry explicit masks: base(x) + s * B(A(x * m / (1 - p_eff)))."""
import numpy as np
import torch

TARGETS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
_MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised Philox4x32-10 (Salmon et al., SC 2011).  Counter words: uint32 arrays (broadcastable); key: two ints."""
    c = [np.asarray(x, dtype=np.uint64) & _MASK32 for x in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0 & 0xFFFFFFFF), np.uint64(k1 & 0xFFFFFFFF)
    for i in range(10):
        if i:
            k0 = (k0 + np.uint64(0x9E3779B9)) & _MASK32
            k1 = (k1 + np.uint64(0xBB67AE85)) & _MASK32
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK32]
    return [x.astype(np.uint32) for x in c]


def threshold(p: float) -> int:
    return int(round(p * 65536))


def keep_mask(seed: int, pass_id: int, layer: int, proj: int, rows, K: int, T: int) -> np.ndarray:
    """bool [len(rows), K]: element (row, col) of projection `proj`'s input in `layer` survives dropout."""
    rows = np.asarray(rows, dtype=np.uint64)
    ng = (K + 7) // 8
    cg = np.arange(ng, dtype=np.uint64)[None, :]
    w = philox4x32_10(cg, rows[:, None], np.uint64((layer << 3) | proj), np.uint64(pass_id & 0xFFFFFFFF),
                      seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    words = np.stack(w, axis=-1)                                            # [rows, ng, 4]
    halves = np.stack([words & 0xFFFF, words >> 16], axis=-1).reshape(len(rows), ng * 8)   # column 8 g + 2 i + h
    return halves[:, :K] >= T


class OracleMasks:
    """Where the masked oracle gets its masks: mask(layer, proj, n_rows, K) -> [n_rows, K] keep flags of global token rows
    [row0, row0 + n_rows).  `row0` is set by the caller when the oracle runs a slice of the pass (one batch row at a time)."""

    def __init__(self, seed: int, pass_id: int, T: int, mask_fn=None):
        self.seed, self.pass_id, self.T, self.row0 = seed, pass_id, T, 0
        self.inv = 65536.0 / (65536 - T)
        self._fn = mask_fn

    def mask(self, layer, proj, n_rows, K, device):
        if self._fn is not None:
            return self._fn(self, layer, proj, n_rows, K).to(device)
        m = keep_mask(self.seed, self.pass_id, layer, proj, np.arange(self.row0, self.row0 + n_rows), K, self.T)
        return torch.from_numpy(m).to(device)


def mask_oracle(text_model, masks: OracleMasks):
    """Turn every OracleLoraLinear of the (already injected) oracle text model into base(x) + s * B(A(x * m / (1 - p_eff))) with
    its projection's mask, drawn from `masks` for the rows of each call."""
    for li, layer in enumerate(text_model.model.layers):
        for parent, names in ((layer.self_attn, TARGETS[:4]), (layer.mlp, TARGETS[4:])):
            for n in names:
                mod = getattr(parent, n)

                def fwd(x, mod=mod, li=li, j=TARGETS.index(n)):
                    K = x.shape[-1]
                    m = masks.mask(li, j, x.numel() // K, K, x.device).to(x.dtype) * masks.inv
                    return mod.base_layer(x) + mod.lora_B["default"](mod.lora_A["default"](x * m.view(x.shape))) * mod.scaling
                mod.forward = fwd
    return text_model
