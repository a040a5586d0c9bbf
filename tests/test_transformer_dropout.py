"""Dropout of the sm_90a transformer expert: the mask definition (CPU Philox reference) and, on the GPU, the kernels and the
trained expert against fp32 oracles that use the same masks (tools/gpu_attention_check.py)."""
import math

import pytest
import torch

import lah_b200  # noqa
from lah_b200.ops import kernels as K
from lah_b200.runtime.native_executor import draw_dropout_seed


@pytest.mark.parametrize("ctr,key,expected", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, expected):
    """Random123 known-answer vectors of philox4x32-10"""
    assert tuple(int(w) for w in K.philox4x32_10_ref(ctr, key)) == expected


@pytest.mark.parametrize("site", [1, 2, 3])
def test_row_col_mask_sub_block_is_slice_of_full_mask(site):
    seed = 0x1234_5678_9abc_def0
    full = K.dropout_mask_ref((64, 512), 0.1, seed, site)
    rows, cols = torch.arange(13, 47).view(-1, 1), torch.arange(101, 333).view(1, -1)
    assert torch.equal(K.dropout_keep_ref(0.1, seed, site, rows, cols), full[13:47, 101:333])


def test_attention_mask_sub_block_and_transpose():
    seed = 2 ** 63 + 5
    full = K.dropout_mask_ref((2, 3, 64, 96), 0.1, seed, K.SITE_ATTN)
    q, k = torch.arange(5, 41), torch.arange(17, 80)
    sub = K.dropout_keep_ref(0.1, seed, K.SITE_ATTN, 1, 2, q.view(-1, 1), k.view(1, -1))
    assert torch.equal(sub, full[1, 2, 5:41, 17:80])
    # key-major indexing (how the backward kernel holds S^T) gives the transposed mask
    transposed = K.dropout_keep_ref(0.1, seed, K.SITE_ATTN, 1, 2, q.view(1, -1), k.view(-1, 1))
    assert torch.equal(transposed, full[1, 2, 5:41, 17:80].t())


def test_sites_seeds_and_heads_are_independent():
    a = K.dropout_mask_ref((64, 256), 0.5, 11, 1)
    assert not torch.equal(a, K.dropout_mask_ref((64, 256), 0.5, 11, 3))
    assert not torch.equal(a, K.dropout_mask_ref((64, 256), 0.5, 12, 1))
    m = K.dropout_mask_ref((1, 2, 32, 32), 0.5, 11, K.SITE_ATTN)
    assert not torch.equal(m[0, 0], m[0, 1])


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("site", [0, 1, 2, 3])
def test_keep_fraction_within_5_sigma(p, site):
    shape = (1, 2, 256, 512) if site == K.SITE_ATTN else (512, 512)
    keep = K.dropout_mask_ref(shape, p, 987654321, site)
    n = keep.numel()
    assert abs(keep.float().mean().item() - (1 - p)) < 5 * math.sqrt(p * (1 - p) / n)


def test_threshold_resolution():
    """16-bit decisions: the realised drop probability threshold / 65536 is within 2^-16 of p"""
    for p in (0.0, 1e-6, 0.1, 0.25, 0.5, 0.9, 0.999999):
        assert abs(K.dropout_threshold(p) / 65536 - p) <= 2 ** -16
    assert K.dropout_threshold(0.1) == 6554
    with pytest.raises(AssertionError):
        K.dropout_threshold(1.0)


def test_seed_draw_follows_torch_manual_seed():
    torch.manual_seed(3)
    a = [draw_dropout_seed() for _ in range(3)]
    torch.manual_seed(3)
    assert [draw_dropout_seed() for _ in range(3)] == a
    assert len(set(a)) == 3 and all(0 <= s < 2 ** 64 for s in a)


@pytest.mark.gpu
@pytest.mark.parametrize("check", ["check_dropout_mask", "check_attention_dropout", "check_transformer_train_dropout"])
def test_transformer_dropout_kernels_and_expert(check):
    """the device masks equal the CPU definition; attention and the default (dropout 0.1) transformer expert train on the
    sm_90a kernels and match fp32 oracles that apply the same masks"""
    from tools import gpu_attention_check as A
    A.results.clear()
    getattr(A, check)()
    bad = {k: v for k, v in A.results.items() if not v.get("ok")}
    assert A.results and not bad, bad
