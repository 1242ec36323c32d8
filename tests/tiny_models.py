"""Random-init tiny models + an in-memory tokenizer (no Hub access) for the host-logic / pipeline tests."""
import torch
from tokenizers import Tokenizer, models, pre_tokenizers
from transformers import LlamaConfig, LlamaForCausalLM, PreTrainedTokenizerFast, Qwen3Config, Qwen3ForCausalLM

VOCAB = 256


def tiny_llama(dtype=torch.float32, device="cpu", head_dim=16, layers=2, heads=4, kv_heads=2, seed=0):
    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=heads * head_dim, num_attention_heads=heads, num_key_value_heads=kv_heads,
                      head_dim=head_dim, num_hidden_layers=layers, intermediate_size=2 * heads * head_dim,
                      vocab_size=VOCAB, max_position_embeddings=16384, eos_token_id=VOCAB - 1, bos_token_id=1,
                      pad_token_id=0)
    model = LlamaForCausalLM(cfg).to(dtype).to(device).eval()
    model.generation_config.eos_token_id = VOCAB - 1
    return model


def tiny_qwen3(dtype=torch.float32, device="cpu", head_dim=16, layers=2, heads=4, kv_heads=2, seed=0):
    torch.manual_seed(seed)
    cfg = Qwen3Config(hidden_size=heads * head_dim, num_attention_heads=heads, num_key_value_heads=kv_heads,
                      head_dim=head_dim, num_hidden_layers=layers, intermediate_size=2 * heads * head_dim,
                      vocab_size=VOCAB, max_position_embeddings=16384, eos_token_id=VOCAB - 1, bos_token_id=1,
                      pad_token_id=0)
    model = Qwen3ForCausalLM(cfg).to(dtype).to(device).eval()
    model.generation_config.eos_token_id = VOCAB - 1
    return model


def tiny_model(family="llama", attn="sdpa", **kw):
    """tiny_llama / tiny_qwen3 (`kw` as they take it) with the attention implementation `attn`."""
    model = (tiny_llama if family == "llama" else tiny_qwen3)(**kw)
    model.config._attn_implementation = attn
    return model


def distinct_ids(n, seed, batch=2, device="cpu"):
    """`batch` prompts of n distinct token ids: a repeated token gives layer-0 keys of exactly equal norm (RoPE keeps
    norms), i.e. exact score ties that torch.topk and the kernels may legitimately break differently."""
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randperm(250, generator=g)[:n] + 2 for _ in range(batch)]).to(device)


def word_tokenizer():
    vocab = {f"w{i}": i for i in range(2, VOCAB - 1)}
    vocab.update({"<pad>": 0, "<s>": 1, "</s>": VOCAB - 1, "<unk>": VOCAB})
    tok = Tokenizer(models.WordLevel(vocab=vocab, unk_token="<unk>"))
    tok.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    fast = PreTrainedTokenizerFast(tokenizer_object=tok, bos_token="<s>", eos_token="</s>", pad_token="<pad>",
                                   unk_token="<unk>")
    fast.model_max_length = 1 << 20
    return fast


def words(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, VOCAB - 1, (n,), generator=g).tolist()
    return " ".join(f"w{i}" for i in ids)
