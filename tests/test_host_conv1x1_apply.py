"""Argument validation of moco_conv1x1_bn_add_relu_fwd (include/moco_b200.h): rejected before any launch, so no GPU is
needed, and a rejected call counts no launch."""
from moco_b200 import _lib

FAKE = 0x10000                                     # 16-byte aligned, never dereferenced: validation fails first


def _layer(gamma=FAKE, eps=1e-5, running_var=None):
    return _lib.BnLayer(gamma, FAKE, None, running_var, None, 0.1, eps, FAKE, FAKE, None, None)


def test_conv1x1_bn_add_relu_fwd_validates_its_arguments():
    lib = _lib.load()
    ws = max(lib.moco_conv1x1_workspace_bytes(), lib.moco_bn_workspace_bytes())
    before = _lib.launches

    def call(x=FAKE, w=FAKE + 4096, res=FAKE + 8192, y=FAKE + 12288, mask=None, M=1024, cin=64, cout=256,
             layer=None, sc=None, given=0, work=FAKE + 16384, nbytes=ws):
        return lib.moco_conv1x1_bn_add_relu_fwd(x, w, res, y, mask, M, cin, cout,
                                                layer if layer is not None else _layer(), sc, given, work, nbytes,
                                                None)

    for bad in [dict(x=None), dict(w=None), dict(res=None), dict(y=None), dict(layer=_layer(None)),
                dict(layer=_layer(eps=0.0)), dict(layer=_layer(running_var=FAKE)), dict(sc=_layer(None)),
                dict(given=4), dict(work=None), dict(given=_lib.BN_STATS_GIVEN, sc=_layer(), work=None),
                dict(x=FAKE + 8), dict(w=FAKE + 2), dict(res=FAKE + 4), dict(y=FAKE + 8), dict(work=FAKE + 8),
                dict(y=FAKE), dict(y=FAKE + 4096), dict(y=FAKE + 8192),              # y aliasing an input
                dict(mask=FAKE + 12288), dict(mask=FAKE + 8192)]:
        assert call(**bad) == -1, bad
        assert b"moco_conv1x1_bn_add_relu_fwd" in lib.moco_last_error()
    for bad in [dict(M=0), dict(M=1 << 31), dict(cin=32), dict(cin=96), dict(cin=65600), dict(cout=32),
                dict(cout=384), dict(cout=4096)]:
        assert call(**bad) == -2, bad
    assert call(nbytes=ws - 1) == -3
    assert call(nbytes=ws - 1, sc=_layer(), given=_lib.BN_STATS_GIVEN) == -3     # the shortcut's statistics pass
    assert _lib.launches == before
