"""
Expert architectures (the L1 "ops/models" layer of SURVEY.md).

* ``FeedforwardBlock(hid)``: x + Linear(h,4h) -> LayerNorm(4h) -> ReLU -> Linear(4h,4h) -> LayerNorm(4h) -> ReLU ->
  Linear(4h,h).  Parameter names match the reference (``layers.{0,1,3,4,6}.{weight,bias}``) so checkpoints are
  interchangeable (/root/reference/experiments/throughput/layers.py:5-19).
* ``TransformerEncoderLayer(d_model, nhead, dim_feedforward=2048, dropout=0.1)``: post-LN encoder layer with GELU,
  batch-first input ``[B, S, d]`` (/root/reference/experiments/throughput/layers.py:22-51).  Unlike the reference it
  does NOT transpose its input in place, so it does not mutate the caller's tensor and it is trainable through
  ``ExpertBackend.backward`` (the reference's block raises there; SURVEY.md §0.3).  Parameter names are identical
  (``self_attn.in_proj_weight`` ..., ``linear1``, ``linear2``, ``norm1``, ``norm2``).  Its four dropouts (attention
  probabilities, ``dropout1``, ``dropout`` after the GELU, ``dropout2``) act in training mode, which is the mode
  ``ExpertBackend`` runs it in; the sm_90a executor (``runtime/native_executor.py``) implements them with in-kernel
  Philox masks (DESIGN.md §9), so the reference's default ``name_to_block["transformer"]`` trains natively.  Like
  ``nn.MultiheadAttention`` it takes any sequence length; the sm_90a executor runs 1 <= S <= ``kernels.MAX_SEQ`` (65536)
  and head dims ``d_model / nhead`` in ``kernels.HEAD_DIMS`` = (32, 64, 128), so ``name_to_block["transformer"](hid_dim)``
  (nhead 16) trains natively at hid_dim 512, 1024 and 2048.  ``causal=True`` makes it a causal (decoder-style) layer:
  position t attends to positions <= t, through an upper-triangular -inf [S, S] ``attn_mask``, which is what
  ``nn.TransformerEncoderLayer`` computes with ``is_causal=True`` and its square subsequent mask; the sm_90a executor
  runs it on the causal attention kernels.  ``causal=False`` (the default) is the reference's layer.
* ``GatedFeedforwardBlock(hid, inner_dim=0, eps=1e-6)``: x + w2(silu(w1(h)) * w3(h)), h = RMSNorm(x), no biases: the
  SwiGLU expert MLP of today's MoE models (parameter names of a Mixtral expert), ``name_to_block["swiglu"]``.

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


#: the parameters of a FeedforwardBlock, in ``parameters()`` order: the segment name the sm_90a code knows each by -> its
#: state_dict key (the reference's names, layers.py:8-16)
FFN_SEG_KEYS = {"w1": "layers.0.weight", "b1": "layers.0.bias", "g1": "layers.1.weight", "be1": "layers.1.bias",
                "w2": "layers.3.weight", "b2": "layers.3.bias", "g2": "layers.4.weight", "be2": "layers.4.bias",
                "w3": "layers.6.weight", "b3": "layers.6.bias"}
FFN_SEG_NAMES = tuple(FFN_SEG_KEYS)
#: bit s set: segment s is a bias or LayerNorm vector (the weight matrices are stepped by the fused wgrad + Adam kernel)
FFN_SMALL_SEG_MASK = sum(1 << s for s, n in enumerate(FFN_SEG_NAMES) if not n.startswith("w"))


class ExpertLayout:
    """How the DMoE engine (``parallel/engine.py``) keeps one expert kind in its flat ``[slots, *shape]`` segments.

    * ``keys``: segment -> the module's state_dict keys it holds, stacked by rows (``[W1; W3]`` is one segment, so the two
      matrices are contiguous per expert and take one GEMM, one dgrad and one fused wgrad + AMSGrad launch);
    * ``params``: the module's parameter keys in ``parameters()`` order (the indices of its optimizer state);
    * ``shapes(hidden, inner)``: segment -> per-expert shape, in segment order;
    * ``small_mask``: bit s set = segment s is a vector (norm / bias), stepped by ``adam_step``, pulled from fp32 into
      shadow slots, zeroed before a shadow gradient reduce; the matrices are stepped by the fused wgrad + AMSGrad kernel;
    * ``buffers(hidden, inner)``: the engine's bf16 row buffers of the kind (see ``LayerWorkspace``).
    """

    def __init__(self, keys, params, shapes, buffers):
        self.keys = dict(keys)
        self.names = tuple(self.keys)
        self.params = tuple(params)
        self.shapes = shapes
        self.buffers = buffers
        self.small_mask = sum(1 << s for s, n in enumerate(self.names) if not n.startswith("w"))
        # parameter key -> (segment, row block, blocks in the segment)
        self.slices = {key: (n, i, len(ks)) for n, ks in self.keys.items() for i, key in enumerate(ks)}
        assert sorted(self.slices) == sorted(self.params)

    def module_state(self, segments):
        """segment -> tensor of one expert  =>  the module's state_dict (in ``params`` order)"""
        out = {}
        for key in self.params:
            n, i, parts = self.slices[key]
            out[key] = segments[n].chunk(parts, 0)[i] if parts > 1 else segments[n]
        return out

    def segment_state(self, state, prefix=""):
        """a module's state_dict  =>  segment -> tensor of one expert (row blocks joined)"""
        return {n: torch.cat([state[prefix + k] for k in ks], 0) if len(ks) > 1 else state[prefix + ks[0]]
                for n, ks in self.keys.items()}


# buffers(H, I): "rows": bf16 [rows, width] activations kept per layer until the backward; "stats": fp32 [rows] per layer;
# "scratch": bf16 [rows, width] backward temporaries shared by all layers; "per_layer": backward buffers read by the fused
# wgrad + AMSGrad launches of the optimizer stream, per layer when that stream is used (else the scratch buffer named)
FFN_LAYOUT = ExpertLayout(
    keys={n: (k,) for n, k in FFN_SEG_KEYS.items()}, params=tuple(FFN_SEG_KEYS.values()),
    shapes=lambda H, I: {"w1": (I, H), "b1": (I,), "g1": (I,), "be1": (I,), "w2": (I, I), "b2": (I,), "g2": (I,),
                         "be2": (I,), "w3": (H, I), "b3": (H,)},
    buffers=lambda H, I: dict(rows={"h1": I, "a1": I, "h2": I, "a2": I}, stats=("mean1", "rstd1", "mean2", "rstd2"),
                              scratch={"da": I, "dh": I}, per_layer={"dh2": "dh", "dh1": "dh"}))
assert FFN_LAYOUT.names == FFN_SEG_NAMES and FFN_LAYOUT.small_mask == FFN_SMALL_SEG_MASK

#: GatedFeedforwardBlock in the engine: the RMSNorm weight, [W1; W3] ([2 inner, hid]: W1 rows [0, inner), W3 rows
#: [inner, 2 inner)) and W2; the keys and parameter order are a Mixtral expert's
GATED_LAYOUT = ExpertLayout(
    keys={"g": ("norm.weight",), "w13": ("w1.weight", "w3.weight"), "w2": ("w2.weight",)},
    params=("norm.weight", "w1.weight", "w2.weight", "w3.weight"),
    shapes=lambda H, I: {"g": (H,), "w13": (2 * I, H), "w2": (H, I)},
    buffers=lambda H, I: dict(rows={"n": H, "h": 2 * I, "a": I}, stats=("rstd",),
                              scratch={"da": I, "dh": 2 * I, "dn": H}, per_layer={"dh13": "dh"}))

#: the layout of every expert kind the engine trains, by its ``name_to_block`` key
EXPERT_LAYOUTS = {"ffn": FFN_LAYOUT, "swiglu": GATED_LAYOUT}


def gated_inner_dim(hid_dim: int) -> int:
    """the default inner width of GatedFeedforwardBlock: 8 hid / 3 rounded up to a multiple of 128 (Llama's convention;
    2816 at hid 1024, 11008 at hid 4096), the parameter count of a 4 hid MLP"""
    return -(-8 * hid_dim // (3 * 128)) * 128


class GatedFeedforwardBlock(nn.Module):
    """
    The gated (SwiGLU) expert MLP of Mixtral, DeepSeek-MoE, Qwen-MoE and Llama, with its RMSNorm pre-norm and residual:
    ``x + w2(silu(w1(h)) * w3(h))``, ``h = norm(x)``.  No biases.  Parameter names ``norm.weight``, ``w1.weight``,
    ``w2.weight``, ``w3.weight`` are those of a Mixtral expert.  ``inner_dim = 0`` selects ``gated_inner_dim(hid_dim)``.
    """

    def __init__(self, hid_dim: int, inner_dim: int = 0, eps: float = 1e-6):
        super().__init__()
        inner = inner_dim or gated_inner_dim(hid_dim)
        self.norm = nn.RMSNorm(hid_dim, eps=eps)
        self.w1 = nn.Linear(hid_dim, inner, bias=False)
        self.w2 = nn.Linear(inner, hid_dim, bias=False)
        self.w3 = nn.Linear(hid_dim, inner, bias=False)

    def forward(self, x):
        h = self.norm(x)
        return x + self.w2(F.silu(self.w1(h)) * self.w3(h))


class TransformerEncoderLayer(nn.Module):
    def __init__(self, d_model: int, nhead: int, dim_feedforward: int = 2048, dropout: float = 0.1, causal: bool = False):
        super().__init__()
        self.causal = causal
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
        if self.causal:   # position t attends to positions <= t
            S = x.shape[0]
            mask = torch.triu(torch.full((S, S), float("-inf"), dtype=x.dtype, device=x.device), diagonal=1)
            attn = self.self_attn(x, x, x, attn_mask=mask, need_weights=False)[0]
        else:
            attn = self.self_attn(x, x, x, need_weights=False)[0]
        x = self.norm1(x + self.dropout1(attn))
        ff = self.linear2(self.dropout(self.activation(self.linear1(x))))
        x = self.norm2(x + self.dropout2(ff))
        return x.transpose(0, 1)


SEQ_LEN = 512  # input shape of the throughput experiment (reference layers.py:57); the layer itself takes any length

name_to_block = {
    "ffn": lambda hid_dim: FeedforwardBlock(hid_dim),
    "transformer": lambda hid_dim: TransformerEncoderLayer(hid_dim, nhead=16),
    "swiglu": lambda hid_dim: GatedFeedforwardBlock(hid_dim),
}
name_to_input = {
    "ffn": lambda batch_size, hid_dim: torch.empty((batch_size, hid_dim)),
    "swiglu": lambda batch_size, hid_dim: torch.empty((batch_size, hid_dim)),
    "transformer": lambda batch_size, hid_dim: torch.empty((batch_size, SEQ_LEN, hid_dim)),
}
