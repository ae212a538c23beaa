"""Offline reward-model fixtures: a random-init Qwen3ForSequenceClassification of a registry shape and a word-level tokenizer built in
memory, saved to a directory that AutoModelForSequenceClassification / AutoTokenizer.from_pretrained load without network access."""
import torch

CHAT_TEMPLATE = "{% for m in messages %}<{{ m['role'] }}> {{ m['content'] }}\n{% endfor %}"


def make_tokenizer(n_words=900, pad=True, chat_template=True):
    """PreTrainedTokenizerFast over ids [UNK]=0, <eos>=1, (<pad>=2), then w0, w1, ... (whitespace-split words)."""
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    special = ["[UNK]", "<eos>"] + (["<pad>"] if pad else [])
    vocab = {t: i for i, t in enumerate(special)}
    vocab.update({f"w{i}": len(special) + i for i in range(n_words)})
    tk = Tokenizer(models.WordLevel(vocab=vocab, unk_token="[UNK]"))
    tk.pre_tokenizer = pre_tokenizers.Whitespace()
    kw = dict(pad_token="<pad>") if pad else {}
    tok = PreTrainedTokenizerFast(tokenizer_object=tk, unk_token="[UNK]", eos_token="<eos>", **kw)
    if chat_template:
        tok.chat_template = CHAT_TEMPLATE
    return tok


def make_reward_model(name="tiny", seed=0, pad_token_id=2):
    """Random-init Qwen3ForSequenceClassification (num_labels = 1) of configs.text_config(name), fp32 on the CPU.  The score head is
    drawn with std d^-1/2, so the rewards spread over about one unit rather than sitting near 0."""
    from transformers import Qwen3ForSequenceClassification
    from bioreason_b200.configs import text_config
    cfg = text_config(name)
    cfg.num_labels = 1
    cfg.pad_token_id = pad_token_id
    torch.manual_seed(seed)
    m = Qwen3ForSequenceClassification(cfg).eval()
    with torch.no_grad():
        m.score.weight.normal_(0.0, cfg.hidden_size ** -0.5)
    return m


def save_reward_dir(path, name="tiny", seed=0, pad=True):
    """Write a reward model and its tokenizer to `path`; returns the path as a string."""
    path = str(path)
    make_reward_model(name, seed).save_pretrained(path)
    make_tokenizer(pad=pad).save_pretrained(path)
    return path
