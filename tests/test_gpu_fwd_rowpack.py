"""GPU tests of the pooled forward on row-packed tiles (even H and W <= 64: several image-row pairs per tile)."""
import pytest
import torch
import torch.nn.functional as F

from hefl_b200 import _ext

pytestmark = pytest.mark.gpu
ops = _ext.ops()


def _fwd_pool(x, wf, b, B, H, W, CK, Co):
    Hp, Wp = (H - 2) // 2, (W - 2) // 2
    out = torch.zeros(B * Hp * Wp, Co, dtype=torch.bfloat16, device="cuda")
    am = torch.full((B * Hp * Wp, Co), 255, dtype=torch.uint8, device="cuda")
    ops.conv_fwd_pool(x.reshape(-1, CK), wf, b, out, am, B, H, W, CK, Co)
    return out, am


# (5, 30) and (3, 62): tiles straddle two images and the last tile is partial; (7, 6, .., 128) and (3, 12, .., 64)
# split the output channels over blockIdx.y; (2, 64) fills all 128 GEMM rows of a tile
@pytest.mark.parametrize("B,H,Ci,CK,Co", [(5, 30, 32, 32, 64), (3, 62, 32, 32, 32), (7, 6, 64, 64, 128),
                                          (3, 12, 64, 64, 64), (2, 64, 32, 32, 32), (3, 14, 32, 32, 64)])
def test_row_packed_forward_matches_torch_and_column_tiles(B, H, Ci, CK, Co):
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.zeros(B, H, H, CK, device="cuda")
    x[..., :Ci] = torch.randn(B, H, H, Ci, device="cuda", generator=g)
    x = x.to(torch.bfloat16)
    w = (torch.randn(Co, Ci, 3, 3, device="cuda", generator=g) * (1.0 / (3 * Ci ** 0.5))).to(torch.bfloat16)
    b = torch.randn(Co, device="cuda", generator=g) * 0.1
    wf = torch.zeros(9, Co, CK, dtype=torch.bfloat16, device="cuda")
    wf[:, :, :Ci] = w.permute(2, 3, 0, 1).reshape(9, Co, Ci)
    Hp = (H - 2) // 2
    out, am = _fwd_pool(x, wf, b, B, H, H, CK, Co)
    # one zero column on the right makes the width odd: the same pooled outputs from the 2 x 128 column tiles
    xpad = torch.zeros(B, H, H + 1, CK, dtype=torch.bfloat16, device="cuda")
    xpad[:, :, :H] = x
    out_c, am_c = _fwd_pool(xpad, wf, b, B, H, H + 1, CK, Co)
    torch.cuda.synchronize()
    # every output gets the same MMAs in the same order on either tiling
    assert torch.equal(out, out_c)
    assert torch.equal(am, am_c)
    xr = x[..., :Ci].float().permute(0, 3, 1, 2)
    ref, idx = F.max_pool2d(F.relu(F.conv2d(xr, w.float(), b)), 2, return_indices=True)
    got = out.view(B, Hp, Hp, Co).permute(0, 3, 1, 2).float()
    assert (got - ref).abs().max() <= 0.02 * ref.abs().max() + 1e-2
    Wo = H - 2
    pos_ref = ((idx // Wo) % 2) * 2 + (idx % Wo) % 2
    code = am.view(B, Hp, Hp, Co).permute(0, 3, 1, 2).long()
    sel = ref > 0.05
    assert ((code & 3)[sel] == pos_ref[sel]).float().mean() > 0.995
    assert torch.equal((code & 4) != 0, got > 0)
    assert int((code & ~7).abs().sum()) == 0          # every pooled output was written
