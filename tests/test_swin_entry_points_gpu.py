"""GPU: the Swin entry points outside the multi-crop forward run the training forward itself (SwinTransformer._run on one
resolution group), so they compute bit for bit what forward([x]) computes, DropPath draws included."""
from functools import partial

import pytest
import torch
import torch.nn as nn

from oracle import golden as GD
from oracle import swin as S

pytestmark = pytest.mark.gpu

ARCHS = {"swin_t_w7": S.SWIN_T_W7, "swin_b_w14": S.SWIN_B_W14}


def _model(spec, drop_path_rate=0.0):
    """CUDA Swin backbone at 224² (num_classes = 0: head = Identity) with seeded non-trivial weights"""
    from esvit_b200.swin_transformer import SwinTransformer
    m = SwinTransformer(img_size=224, num_classes=0, drop_path_rate=drop_path_rate,
                        norm_layer=partial(nn.LayerNorm, eps=1e-6), **spec)
    m.load_state_dict(GD.seeded_state_dict(GD.recipe(m.state_dict()), 7))
    return m.cuda()


def _images():
    return torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(12)).cuda()


@pytest.mark.parametrize("arch", list(ARCHS))
def test_n_last_blocks_1_equals_forward(arch):
    spec = dict(ARCHS[arch])
    m = _model(spec).eval()
    x = _images()
    with torch.no_grad():
        f = m(x)
        f1 = m.forward_return_n_last_blocks(x, 1, False, list(spec["depths"]))
    assert torch.equal(f1, f)


@pytest.mark.parametrize("arch", list(ARCHS))
def test_forward_features_with_drop_path_equals_forward(arch):
    m = _model(dict(ARCHS[arch]), drop_path_rate=0.2).train()
    x = _images()
    with torch.no_grad():
        torch.manual_seed(3)
        a = m.forward_features(x)
        torch.manual_seed(3)
        b = m([x])
        torch.manual_seed(4)
        c = m([x])
    assert torch.equal(a, b)
    assert not torch.equal(b, c)  # DropPath is active: another draw gives another result
