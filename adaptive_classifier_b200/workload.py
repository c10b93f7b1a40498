"""Synthetic workloads of BASELINE.json / SURVEY.md section 8(d), shared by bench.py, __graft_entry__.smoke() and tests.

No network, no datasets, no checkpoints: seeded random-init bert-base architecture, synthetic token ids,
class-structured synthetic prototype rows (row j belongs to class j mod C)."""
from __future__ import annotations

import torch


def bert_base_state_dict(seed: int = 1234, **cfg_over):
    """HF BertModel(BertConfig()) == bert-base-uncased architecture, random init under torch.manual_seed(seed)."""
    from transformers import BertConfig, BertModel
    torch.manual_seed(seed)
    cfg = BertConfig(**cfg_over)
    m = BertModel(cfg, add_pooling_layer=False)
    m.eval()
    return m, cfg


def modernbert_base(seed: int = 1234):
    """HF ModernBertModel(ModernBertConfig()) == ModernBERT-base architecture (22 x 768, 12 heads, GeGLU I = 1152, vocab 50368,
    sliding half-window 64 on two of every three layers), random init under torch.manual_seed(seed)."""
    from transformers import ModernBertConfig, ModernBertModel
    torch.manual_seed(seed)
    cfg = ModernBertConfig()
    m = ModernBertModel(cfg)
    m.eval()
    return m, cfg


def mpnet_base(seed: int = 1234):
    """HF MPNetModel of the sentence-transformers/all-mpnet-base-v2 shape (12 x 768, 12 heads, I = 3072, vocab 30527,
    max_position_embeddings 514, LayerNorm eps 1e-5, 32 relative-attention buckets), random init under
    torch.manual_seed(seed)."""
    from transformers import MPNetConfig, MPNetModel
    torch.manual_seed(seed)
    cfg = MPNetConfig(vocab_size=30527, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                      intermediate_size=3072, max_position_embeddings=514, layer_norm_eps=1e-5)
    m = MPNetModel(cfg, add_pooling_layer=False)
    m.eval()
    return m, cfg


def deberta_base(seed: int = 1234):
    """HF DebertaV2Model of the microsoft/deberta-v3-base shape (12 x 768, 12 heads, I = 3072, vocab 128100, 256 position
    buckets, share_att_key, LayerNorm-ed relative embeddings, no position or token-type table, LayerNorm eps 1e-7), random
    init under torch.manual_seed(seed), with the relative embeddings drawn N(0, 1) (the init's std 0.02 goes through the
    encoder's LayerNorm either way) so that the position terms move the scores."""
    from transformers import DebertaV2Config, DebertaV2Model
    torch.manual_seed(seed)
    cfg = DebertaV2Config(vocab_size=128100, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                          intermediate_size=3072, max_position_embeddings=512, type_vocab_size=0, relative_attention=True,
                          position_buckets=256, norm_rel_ebd="layer_norm", share_att_key=True, pos_att_type=["p2c", "c2p"],
                          position_biased_input=False, layer_norm_eps=1e-7, hidden_act="gelu", pad_token_id=0)
    m = DebertaV2Model(cfg)
    m.eval()
    return m, cfg


def albert_base(seed: int = 1234, large: bool = False):
    """HF AlbertModel of the albert-base-v2 shape (12 x 768, 12 heads, I = 3072, embedding_size 128, vocab 30000, one shared
    layer, "gelu_new"), or with large the albert-large-v2 shape (24 x 1024, 16 heads, I = 4096), random init under
    torch.manual_seed(seed)."""
    from transformers import AlbertConfig, AlbertModel
    torch.manual_seed(seed)
    dims = dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096) if large else \
        dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072)
    cfg = AlbertConfig(vocab_size=30000, embedding_size=128, num_hidden_groups=1, inner_group_num=1, hidden_act="gelu_new",
                       max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12, **dims)
    m = AlbertModel(cfg, add_pooling_layer=False)
    m.eval()
    return m, cfg


def albert_large(seed: int = 1234):
    return albert_base(seed, large=True)


def electra_small(seed: int = 1234):
    """HF ElectraModel of the google/electra-small-discriminator shape (12 x 256, 4 heads, I = 1024, embedding_size 128,
    vocab 30522, "gelu"), random init under torch.manual_seed(seed)."""
    from transformers import ElectraConfig, ElectraModel
    torch.manual_seed(seed)
    cfg = ElectraConfig(vocab_size=30522, embedding_size=128, hidden_size=256, num_hidden_layers=12, num_attention_heads=4,
                        intermediate_size=1024, max_position_embeddings=512, type_vocab_size=2, hidden_act="gelu")
    m = ElectraModel(cfg)
    m.eval()
    return m, cfg


def bge_m3(seed: int = 1234):
    """HF XLMRobertaModel of the BAAI/bge-m3 shape (XLM-RoBERTa-large with 8194 positions: 24 x 1024, 16 heads, I = 4096,
    vocab 250002, pad id 1, one token type, LayerNorm eps 1e-5), random init under torch.manual_seed(seed).
    Snowflake/snowflake-arctic-embed-l-v2.0 has the same shape."""
    from transformers import XLMRobertaConfig, XLMRobertaModel
    torch.manual_seed(seed)
    cfg = XLMRobertaConfig(vocab_size=250002, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                           intermediate_size=4096, max_position_embeddings=8194, type_vocab_size=1, layer_norm_eps=1e-5,
                           pad_token_id=1, bos_token_id=0, eos_token_id=2)
    m = XLMRobertaModel(cfg, add_pooling_layer=False)
    m.eval()
    return m, cfg


def nomic_v15(seed: int = 1234):
    """HF NomicBertModel(NomicBertConfig()) == nomic-ai/nomic-embed-text-v1 / v1.5 architecture (12 x 768, 12 heads, SwiGLU
    I = 3072 without biases, no q/k/v/o biases, RoPE theta 1000, 2048 positions, vocab 30528), random init under
    torch.manual_seed(seed).  Token ids: synthetic_ids(B, S, vocab=30528)."""
    from transformers import NomicBertConfig, NomicBertModel
    torch.manual_seed(seed)
    cfg = NomicBertConfig()
    m = NomicBertModel(cfg)
    m.eval()
    return m, cfg


def jina_v3(seed: int = 1234):
    """HF JinaEmbeddingsV3Model(JinaEmbeddingsV3Config()) == jinaai/jina-embeddings-v3 architecture (24 x 1024, 16 heads,
    GELU I = 4096 with biases, RoPE theta 20000, 8194 positions of which 8192 are used, vocab 250002, one token type), random
    init under torch.manual_seed(seed), without the pooler.  Token ids: xlmr_ids."""
    from transformers import JinaEmbeddingsV3Config, JinaEmbeddingsV3Model
    torch.manual_seed(seed)
    cfg = JinaEmbeddingsV3Config()
    m = JinaEmbeddingsV3Model(cfg, add_pooling_layer=False)
    m.eval()
    return m, cfg


def eurobert_210m(seed: int = 1234):
    """EuroBERT/EuroBERT-210m architecture as HF EuroBertModel (12 x 768, 12 heads of 64 with as many kv heads, SwiGLU
    I = 3072 without biases, RMSNorm eps 1e-5, RoPE theta 250000, 8192 positions, vocab 128256), random init under
    torch.manual_seed(seed).  The hub config cannot be read offline: the dims are those of the EuroBERT paper
    (arXiv:2503.05500) and the model card, and EuroBertConfig()'s defaults for the rest.  Token ids: synthetic_ids(B, S,
    vocab=128256)."""
    from transformers import EuroBertConfig, EuroBertModel
    torch.manual_seed(seed)
    cfg = EuroBertConfig(vocab_size=128256, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                         num_attention_heads=12, num_key_value_heads=12, max_position_embeddings=8192,
                         rope_parameters={"rope_type": "default", "rope_theta": 250000.0})
    m = EuroBertModel(cfg)
    m.eval()
    return m, cfg


def xlmr_ids(B: int, S: int, seed: int = 7, vocab: int = 250002) -> torch.Tensor:
    """uniform in [5, vocab), <s>=0 first, </s>=2 last, never the pad id 1; int32 [B,S] on the host."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(5, vocab, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0], ids[:, -1] = 0, 2
    return ids.to(torch.int32)


def modernbert_ids(B: int, S: int, seed: int = 7) -> torch.Tensor:
    """uniform in [1000, 50000), [CLS]=50281 first, [SEP]=50282 last, never the pad id 50283; int32 [B,S] on the host."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1000, 50000, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0], ids[:, -1] = 50281, 50282
    return ids.to(torch.int32)


def synthetic_ids(B: int, S: int, vocab: int = 30522, seed: int = 7) -> torch.Tensor:
    """uniform in [1000, vocab), [CLS]=101 first, [SEP]=102 last, no padding; int32 [B,S] on the host."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(min(1000, vocab - 1), vocab, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0] = min(101, vocab - 1)
    ids[:, -1] = min(102, vocab - 1)
    return ids.to(torch.int32)


def class_centres(C: int, D: int, device="cpu") -> torch.Tensor:
    g = torch.Generator().manual_seed(0)
    return torch.nn.functional.normalize(torch.randn(C, D, generator=g), dim=1).to(device)


def synthetic_rows(lo: int, hi: int, D: int, C: int, seed: int, device="cuda", chunk: int = 131072) -> torch.Tensor:
    """rows [lo,hi) of the synthetic index: normalize(centre[j mod C] + 0.5*randn/sqrt(D)); generated on `device` in chunks
    with a device generator seeded by (seed, GLOBAL chunk start): any row range of the same index has the same bits, so a row
    shard equals the corresponding slice of the unsharded matrix (the N > 1 parity check of bench.py relies on it)."""
    cen = class_centres(C, D, device)
    out = torch.empty((hi - lo, D), dtype=torch.float32, device=device)
    for s in range(lo - lo % chunk, hi, chunk):
        g = torch.Generator(device=device).manual_seed(seed * 1_000_003 + s)
        noise = torch.randn((chunk, D), generator=g, device=device) * (0.5 / D ** 0.5)
        a, e = max(s, lo), min(hi, s + chunk)
        j = torch.arange(a, e, device=device) % C
        out[a - lo : e - lo] = torch.nn.functional.normalize(cen[j] + noise[a - s : e - s], dim=1)
    return out


def synthetic_queries_embeddings(B: int, D: int, C: int, seed: int = 1, device="cuda") -> torch.Tensor:
    """isolated-kNN queries: same construction around the same centres, query b belongs to class b mod C."""
    cen = class_centres(C, D, device)
    g = torch.Generator(device=device).manual_seed(seed + 777)
    noise = torch.randn((B, D), generator=g, device=device) * (0.5 / D ** 0.5)
    return torch.nn.functional.normalize(cen[torch.arange(B, device=device) % C] + noise, dim=1)
