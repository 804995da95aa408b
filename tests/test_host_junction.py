"""Argument validation of the two-gradient backward entry points moco_bn_add_relu_bwd2 and moco_maxpool3x3s2_bwd2
(include/moco_b200.h): rejected before any launch, so no GPU is needed."""
from moco_b200 import _lib
from moco_b200.bn import BatchNormAct2d, hand_over

FAKE = 0x10000                                     # 16-byte aligned, never dereferenced: validation fails first


def _layer(bwd=True):
    return _lib.BnLayer(FAKE, FAKE, None, None, None, 0.1, 1e-5, FAKE, FAKE, FAKE if bwd else None,
                        FAKE if bwd else None)


def test_bn_add_relu_bwd2_validates_its_arguments():
    lib = _lib.load()
    ws = lib.moco_bn_workspace_bytes()
    before = _lib.launches
    for dy, dy2, layer, extra in [(FAKE, None, _layer(), FAKE), (None, FAKE, _layer(), FAKE),
                                  (FAKE, FAKE + 8, _layer(), FAKE), (FAKE, FAKE, _layer(False), FAKE),
                                  (FAKE, FAKE, _layer(), None)]:
        rc = lib.moco_bn_add_relu_bwd2(dy, dy2, FAKE, FAKE, extra, 1024, 64, layer, None, FAKE, None, FAKE, ws, None)
        assert rc == -1 and b"moco_bn_add_relu_bwd2" in lib.moco_last_error()
    # a shortcut BN needs residual and dresidual
    rc = lib.moco_bn_add_relu_bwd2(FAKE, FAKE, FAKE, None, FAKE, 1024, 64, _layer(), _layer(), FAKE, FAKE, FAKE, ws,
                                   None)
    assert rc == -1
    assert lib.moco_bn_add_relu_bwd2(FAKE, FAKE, FAKE, None, FAKE, 1024, 64, _layer(), None, FAKE, None, FAKE, 16,
                                     None) == -3
    assert _lib.launches == before


def test_maxpool_bwd2_validates_its_arguments():
    lib = _lib.load()
    before = _lib.launches
    for dy, dy2, taps in [(None, FAKE, FAKE), (FAKE, None, FAKE), (FAKE, FAKE + 8, FAKE), (FAKE, FAKE, FAKE + 4)]:
        assert lib.moco_maxpool3x3s2_bwd2(dy, dy2, taps, FAKE, 1, 8, 8, 64, None) == -1
        assert b"moco_maxpool3x3s2_bwd2" in lib.moco_last_error()
    assert lib.moco_maxpool3x3s2_bwd2(FAKE, FAKE, FAKE, FAKE, 1, 8, 8, 12, None) == -2      # C % 8 != 0
    assert lib.moco_maxpool3x3s2_bwd2(FAKE, FAKE, FAKE, FAKE, 70000, 8, 8, 64, None) == -2  # N > 65535
    assert _lib.launches == before


def test_hand_over_passes_cpu_tensors_through():
    import torch
    x = torch.randn(2, 64, 4, 4, requires_grad=True)
    y = BatchNormAct2d(64, relu=True)(x, torch.randn(2, 64, 4, 4))
    assert hand_over(y) is y                       # nn.BatchNorm2d's own path: autograd adds the gradients
