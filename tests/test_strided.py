"""CPU tests of the batch-stride qualification (flashfftconv.conv.batch_stride): which (B, H, L) views the engine reads
and writes in place through bffc_fwd_strided / bffc_bwd_strided, and which are copied to a contiguous tensor first."""
import pytest
import torch

BF16 = torch.bfloat16


@pytest.fixture(scope='module')
def conv():
    import __graft_entry__ as ge
    ge.build()
    from flashfftconv import conv
    return conv


def test_projection_slices_qualify(conv):
    B, D, L = 3, 5, 64
    proj = torch.zeros(B, 3 * D, L, dtype=BF16)
    for t in proj.split(D, dim=1):
        assert conv.batch_stride(t, BF16, 'cpu') == 3 * D * L
    assert conv.batch_stride(proj[:, D:2 * D].contiguous(), BF16, 'cpu') == D * L
    # a batch stride that is a larger multiple of 8 than H*L
    buf = torch.zeros(B, D * L + 8, dtype=BF16)
    assert conv.batch_stride(buf[:, :D * L].view(B, D, L), BF16, 'cpu') == D * L + 8


def test_views_that_do_not_qualify(conv):
    B, D, L = 3, 5, 64
    proj = torch.zeros(B, 3 * D, L, dtype=BF16)
    x1 = proj[:, :D]
    assert conv.batch_stride(x1, BF16) is None                              # not on the device
    assert conv.batch_stride(x1, torch.float16, 'cpu') is None              # wrong dtype
    assert conv.batch_stride(x1.transpose(0, 1), BF16, 'cpu') is None       # channel and batch swapped
    assert conv.batch_stride(x1.transpose(1, 2), BF16, 'cpu') is None       # rows not contiguous
    flat = torch.zeros(B * D * L + 1, dtype=BF16)
    assert conv.batch_stride(flat[1:].view(B, D, L), BF16, 'cpu') is None   # storage offset of one element
    buf = torch.zeros(B, D * L + 4, dtype=BF16)
    assert conv.batch_stride(buf[:, :D * L].view(B, D, L), BF16, 'cpu') is None   # batch stride not a multiple of 8
    overlap = torch.zeros(B * D * L, dtype=BF16).as_strided((B, D, L), ((D - 1) * L, L, 1))
    assert conv.batch_stride(overlap, BF16, 'cpu') is None                  # batch stride < H*L: members overlap
