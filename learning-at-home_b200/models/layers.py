"""
Expert architectures (the L1 "ops/models" layer of SURVEY.md).

* ``FeedforwardBlock(hid)``: x + Linear(h,4h) -> LayerNorm(4h) -> ReLU -> Linear(4h,4h) -> LayerNorm(4h) -> ReLU ->
  Linear(4h,h).  Parameter names match the reference (``layers.{0,1,3,4,6}.{weight,bias}``) so checkpoints are
  interchangeable (/root/reference/experiments/throughput/layers.py:5-19).
* ``TransformerEncoderLayer(d_model, nhead, dim_feedforward=2048, dropout=0.1)``: post-LN encoder layer with GELU,
  batch-first input ``[B, S, d]`` (/root/reference/experiments/throughput/layers.py:22-51).  Unlike the reference it
  does NOT transpose its input in place, so it does not mutate the caller's tensor and it is trainable through
  ``ExpertBackend.backward`` (the reference's block raises there; SURVEY.md §0.3).  Parameter names are identical
  (``self_attn.in_proj_weight`` ..., ``linear1``, ``linear2``, ``norm1``, ``norm2``).

These are the plain PyTorch definitions (CPU path, oracle, checkpoint container).  The sm_90a execution of the same
maths lives in ``lah_b200.parallel.engine`` (grouped wgmma GEMMs + fused LN/ReLU/Adam kernels).
"""
import torch
from torch import nn
import torch.nn.functional as F


class FeedforwardBlock(nn.Module):
    def __init__(self, hid_dim: int):
        super().__init__()
        inner = 4 * hid_dim
        self.layers = nn.Sequential(
            nn.Linear(hid_dim, inner),      # 0
            nn.LayerNorm(inner),            # 1
            nn.ReLU(),                      # 2
            nn.Linear(inner, inner),        # 3
            nn.LayerNorm(inner),            # 4
            nn.ReLU(),                      # 5
            nn.Linear(inner, hid_dim),      # 6
        )

    def forward(self, x):
        return x + self.layers(x)


class TransformerEncoderLayer(nn.Module):
    def __init__(self, d_model: int, nhead: int, dim_feedforward: int = 2048, dropout: float = 0.1):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)
        self.dropout1 = nn.Dropout(dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.activation = nn.GELU()

    def forward(self, src):
        # src: [batch, seq, d_model]; attention runs sequence-first on a transposed VIEW (no in-place transpose)
        x = src.transpose(0, 1)
        attn = self.self_attn(x, x, x, need_weights=False)[0]
        x = self.norm1(x + self.dropout1(attn))
        ff = self.linear2(self.dropout(self.activation(self.linear1(x))))
        x = self.norm2(x + self.dropout2(ff))
        return x.transpose(0, 1)


SEQ_LEN = 512  # the throughput experiment hard-codes 512-token sequences (reference layers.py:57)

name_to_block = {
    "ffn": lambda hid_dim: FeedforwardBlock(hid_dim),
    "transformer": lambda hid_dim: TransformerEncoderLayer(hid_dim, nhead=16),
}
name_to_input = {
    "ffn": lambda batch_size, hid_dim: torch.empty((batch_size, hid_dim)),
    "transformer": lambda batch_size, hid_dim: torch.empty((batch_size, SEQ_LEN, hid_dim)),
}
