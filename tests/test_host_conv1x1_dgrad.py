"""Argument validation of moco_conv1x1_dgrad_bn_bwd and moco_bn_bwd_apply_given (include/moco_b200.h): rejected before
any launch, so no GPU is needed."""
from moco_b200 import _lib

FAKE = 0x10000                                     # 16-byte aligned, never dereferenced: validation fails first


def _layer(dgamma=FAKE):
    return _lib.BnLayer(FAKE, None, None, None, None, 0.0, 0.0, FAKE, FAKE, dgamma, FAKE)


def test_conv1x1_dgrad_bn_bwd_validates_its_arguments():
    lib = _lib.load()
    ws = lib.moco_conv1x1_workspace_bytes()
    before = _lib.launches

    def call(dh=FAKE, w=FAKE + 4096, g=FAKE + 8192, M=1024, cin=256, cout=64, x=FAKE + 12288, mask=FAKE + 16384,
             dy2=FAKE + 20480, x2=None, layer=None, sc=None, work=FAKE + 24576, nbytes=ws):
        return lib.moco_conv1x1_dgrad_bn_bwd(dh, w, g, M, cin, cout, x, mask, dy2, x2,
                                             layer if layer is not None else _layer(), sc, work, nbytes, None)

    for bad in [dict(dh=None), dict(w=None), dict(g=None), dict(x=None), dict(work=None), dict(layer=_layer(None)),
                dict(dh=FAKE + 8), dict(w=FAKE + 2), dict(g=FAKE + 4), dict(x=FAKE + 8), dict(mask=FAKE + 1),
                dict(dy2=FAKE + 8), dict(work=FAKE + 8), dict(g=FAKE), dict(g=FAKE + 12288), dict(g=FAKE + 20480),
                dict(g=FAKE + 4096), dict(g=FAKE + 16384),           # g aliasing w or the mask bytes
                dict(x2=FAKE + 28672),                               # x2 without the shortcut BN
                dict(sc=_layer())]:                                  # and the reverse
        assert call(**bad) == -1, bad
        assert b"moco_conv1x1_dgrad_bn_bwd" in lib.moco_last_error()
    for bad in [dict(M=0), dict(M=1 << 31), dict(cin=64), dict(cin=384), dict(cin=4096), dict(cout=32),
                dict(cout=96), dict(cout=4160), dict(mask=None), dict(dy2=None),
                dict(x2=FAKE + 28672, sc=_layer())]:                 # a downsample block's bn3: not implemented
        assert call(**bad) == -2, bad
    assert call(nbytes=ws - 1) == -3
    assert _lib.launches == before


def test_bn_bwd_apply_given_validates_its_arguments():
    lib = _lib.load()
    before = _lib.launches

    def call(g=FAKE, x=FAKE + 4096, x2=None, M=1024, C=64, layer=None, sc=None, dx=FAKE + 8192, dx2=None):
        return lib.moco_bn_bwd_apply_given(g, x, x2, M, C, layer if layer is not None else _layer(), sc, dx, dx2,
                                           None)

    for bad in [dict(g=None), dict(x=None), dict(dx=None), dict(layer=_layer(None)), dict(g=FAKE + 8),
                dict(x=FAKE + 2), dict(dx=FAKE + 4), dict(sc=_layer()), dict(sc=_layer(), x2=FAKE + 12288),
                dict(sc=_layer(None), x2=FAKE + 12288, dx2=FAKE + 16384),
                dict(sc=_layer(), x2=FAKE + 12292, dx2=FAKE + 16384)]:
        assert call(**bad) == -1, bad
        assert b"moco_bn_bwd_apply_given" in lib.moco_last_error()
    for bad in [dict(M=0), dict(C=96), dict(C=32), dict(C=4096),
                dict(sc=_layer(), x2=FAKE + 12288, dx2=FAKE + 16384)]:      # a shortcut BN: not implemented
        assert call(**bad) == -2, bad
    assert _lib.launches == before
