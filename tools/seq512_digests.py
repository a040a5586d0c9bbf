"""SHA-256 digests of what the transformer expert's kernels compute on 512-token sequences: attention forward (output and
log-sum-exp) and backward at p = 0 and p = 0.1, the site-0 dropout mask, and one seeded ExpertBackend.backward of the
default expert (dropout 0.1): dL/dx and every updated parameter.  All inputs come from fixed seeds on the CPU.

tests/golden/seq512_digests.json holds the digests of the kernels that only ran S = 512; tests/test_transformer_seq_len.py
recomputes them, so a change of a single bit at S = 512 fails there.

    python tools/seq512_digests.py OUT.json      # needs a GPU; computes everything twice and checks it is repeatable
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import lah_b200  # noqa

SEED = 0x5EED0512


def sha(*tensors):
    h = hashlib.sha256()
    for t in tensors:
        t = t.detach().contiguous().cpu()
        h.update(f"{t.dtype}{tuple(t.shape)}".encode())
        h.update(t.reshape(-1).view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


def compute():
    from lah_b200 import BatchTensorProto, ExpertBackend
    from lah_b200.models.layers import name_to_block
    from lah_b200.ops import kernels as K
    out = {}
    gen = torch.Generator().manual_seed(512)
    batch, heads, d = 2, 16, 1024
    T = batch * 512
    qkv = (torch.randn(T, 3 * d, generator=gen) * 1.2).to(torch.bfloat16).cuda()
    dout = torch.randn(T, d, generator=gen).to(torch.bfloat16).cuda()
    for p in (0.0, 0.1):
        drop = (p, SEED) if p else None
        lse = torch.empty(T, heads, device="cuda")
        o = K.attention_fwd(qkv, heads, lse=lse, dropout=drop)
        dqkv = K.attention_bwd(qkv, o, dout, lse, heads, dropout=drop)
        out[f"attention_fwd_p{p}"] = sha(o, lse)
        out[f"attention_bwd_p{p}"] = sha(dqkv)
    out["dropout_mask_1x2x512x512"] = sha(K.dropout_mask((1, 2, 512, 512), 0.1, SEED, K.SITE_ATTN))

    torch.manual_seed(0)
    layer = name_to_block["transformer"](1024)
    x = torch.randn(2, 512, 1024, generator=gen)
    g = torch.randn(2, 512, 1024, generator=gen) * 0.1
    layer.cuda()
    be = ExpertBackend(name="t", expert=layer, opt=torch.optim.Adam(layer.parameters(), lr=1e-4, amsgrad=True),
                       args_schema=(BatchTensorProto(512, 1024),), outputs_schema=BatchTensorProto(512, 1024),
                       max_batch_size=8)
    torch.manual_seed(7)   # the executor draws its dropout seed from torch's CPU generator
    (dx,) = be.backward(x.cuda(), g.cuda())
    assert type(be._executor).__name__ == "NativeTransformerExecutor", be._executor
    out["expert_backward_dx"] = sha(dx)
    out["expert_backward_params"] = sha(*[v for _, v in sorted(be.state_dict().items())])
    torch.cuda.synchronize()
    return out


if __name__ == "__main__":
    first, second = compute(), compute()
    assert first == second, "the digests are not repeatable"
    with open(sys.argv[1], "w") as f:
        json.dump(first, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(first, indent=1, sort_keys=True))
