"""BERT-base with the pre-training heads (110,106,428 parameters) -- the BASELINE "Keras BERT-base
Horovod-path" configuration.  Not in the reference tree; it exercises the all-reduce path at
220 MB (bf16) of gradients per step (SURVEY.md §2.5).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn as nn
import torch.nn.functional as F

N_PARAMS = 110_106_428


class BertLayer(nn.Module):
    def __init__(self, hidden: int, heads: int, intermediate: int, dropout: float):
        super().__init__()
        self.heads = heads
        self.qkv = nn.Linear(hidden, 3 * hidden)
        self.out = nn.Linear(hidden, hidden)
        self.ln1 = nn.LayerNorm(hidden, eps=1e-12)
        self.ffn1 = nn.Linear(hidden, intermediate)
        self.ffn2 = nn.Linear(intermediate, hidden)
        self.ln2 = nn.LayerNorm(hidden, eps=1e-12)
        self.drop = dropout

    def forward(self, x, mask):
        B, S, H = x.shape
        q, k, v = self.qkv(x).view(B, S, 3, self.heads, H // self.heads).permute(2, 0, 3, 1, 4)
        a = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=self.drop if self.training else 0.0)
        a = a.transpose(1, 2).reshape(B, S, H)
        x = self.ln1(x + F.dropout(self.out(a), self.drop, self.training))
        h = self.ffn2(F.gelu(self.ffn1(x)))
        return self.ln2(x + F.dropout(h, self.drop, self.training))


class BertForPreTraining(nn.Module):
    def __init__(self, vocab: int = 30522, hidden: int = 768, layers: int = 12, heads: int = 12,
                 intermediate: int = 3072, max_pos: int = 512, type_vocab: int = 2, dropout: float = 0.1):
        super().__init__()
        self.word = nn.Embedding(vocab, hidden)
        self.pos = nn.Embedding(max_pos, hidden)
        self.typ = nn.Embedding(type_vocab, hidden)
        self.emb_ln = nn.LayerNorm(hidden, eps=1e-12)
        self.layers = nn.ModuleList([BertLayer(hidden, heads, intermediate, dropout) for _ in range(layers)])
        self.pooler = nn.Linear(hidden, hidden)
        self.mlm_dense = nn.Linear(hidden, hidden)
        self.mlm_ln = nn.LayerNorm(hidden, eps=1e-12)
        self.mlm_bias = nn.Parameter(torch.zeros(vocab))
        self.nsp = nn.Linear(hidden, 2)
        self.drop = dropout
        self.apply(self._init)

    @staticmethod
    def _init(m):
        if isinstance(m, (nn.Linear, nn.Embedding)):
            nn.init.normal_(m.weight, std=0.02)
            if isinstance(m, nn.Linear) and m.bias is not None:
                nn.init.zeros_(m.bias)

    def forward(self, inputs: Dict[str, torch.Tensor]):
        ids = inputs["input_ids"]
        B, S = ids.shape
        pos = torch.arange(S, device=ids.device).unsqueeze(0)
        x = self.word(ids) + self.pos(pos) + self.typ(inputs["token_type_ids"])
        x = F.dropout(self.emb_ln(x), self.drop, self.training)
        mask = None
        if "attention_mask" in inputs:
            mask = inputs["attention_mask"][:, None, None, :].to(torch.bool)
        for layer in self.layers:
            x = layer(x, mask)
        pooled = torch.tanh(self.pooler(x[:, 0]))
        h = self.mlm_ln(F.gelu(self.mlm_dense(x)))
        mlm_logits = F.linear(h, self.word.weight, self.mlm_bias)        # decoder tied to the embeddings
        return {"mlm_logits": mlm_logits, "nsp_logits": self.nsp(pooled)}


def pretraining_loss(y: Dict[str, torch.Tensor], out: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Masked-LM cross-entropy (labels == -100 ignored) + next-sentence cross-entropy."""
    mlm = F.cross_entropy(out["mlm_logits"].float().flatten(0, 1), y["mlm_labels"].flatten(), ignore_index=-100)
    nsp = F.cross_entropy(out["nsp_logits"].float(), y["nsp_labels"])
    return mlm + nsp


def synthetic_batch(batch: int, seq_len: int = 128, vocab: int = 30522, seed: int = 0, mask_rate: float = 0.15):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1000, vocab, (batch, seq_len), generator=g)
    types = (torch.arange(seq_len)[None, :] >= seq_len // 2).long().expand(batch, seq_len).contiguous()
    labels = torch.full((batch, seq_len), -100, dtype=torch.long)
    masked = torch.rand(batch, seq_len, generator=g) < mask_rate
    labels[masked] = ids[masked]
    ids = ids.clone()
    ids[masked] = 103
    x = {"input_ids": ids, "token_type_ids": types}
    y = {"mlm_labels": labels, "nsp_labels": torch.randint(0, 2, (batch,), generator=g)}
    return x, y


def keras_bert_base(**kwargs):
    """BERT-base as a mini-Keras model (trains through the H100 graph engine + fused K4 Adam step)."""
    from tf_yarn_b200 import keras
    return keras.Model.from_torch(BertForPreTraining(**kwargs), name="bert_base")
