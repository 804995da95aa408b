"""Argument validation of moco_conv1x1_bn_stats and moco_bn_fwd_train_given (include/moco_b200.h): rejected before any
launch, so no GPU is needed."""
from moco_b200 import _lib

FAKE = 0x10000                                     # 16-byte aligned, never dereferenced: validation fails first


def _layer(eps=1e-5):
    return _lib.BnLayer(FAKE, FAKE, None, None, None, 0.1, eps, FAKE, FAKE, None, None)


def test_conv1x1_bn_stats_validates_its_arguments():
    lib = _lib.load()
    ws = lib.moco_conv1x1_workspace_bytes()
    before = _lib.launches
    call = lambda x=FAKE, w=FAKE, y=FAKE + 4096, M=1024, cin=64, cout=64, layer=None, work=FAKE, nbytes=ws: \
        lib.moco_conv1x1_bn_stats(x, w, y, M, cin, cout, layer if layer is not None else _layer(), work, nbytes, None)
    for bad in [dict(x=None), dict(w=None), dict(y=None), dict(work=None), dict(x=FAKE + 8), dict(w=FAKE + 2),
                dict(y=FAKE + 4), dict(work=FAKE + 8), dict(y=FAKE), dict(layer=_layer(eps=0.0))]:
        assert call(**bad) == -1, bad
        assert b"moco_conv1x1_bn_stats" in lib.moco_last_error()
    for bad in [dict(M=0), dict(cin=96), dict(cout=32), dict(cin=0), dict(cout=4160), dict(M=1 << 31)]:
        assert call(**bad) == -2, bad
    assert call(nbytes=ws - 1) == -3
    assert _lib.launches == before


def test_bn_fwd_train_given_validates_its_arguments():
    lib = _lib.load()
    ws = lib.moco_bn_workspace_bytes()
    G, SG = _lib.BN_STATS_GIVEN, _lib.BN_SC_STATS_GIVEN
    before = _lib.launches
    call = lambda x=FAKE, r=None, y=FAKE + 4096, sc=None, given=G, work=None, nbytes=0, C=64: \
        lib.moco_bn_fwd_train_given(x, r, y, None, 1024, C, 1, _layer(), sc, given, work, nbytes, None)
    for bad in [dict(x=None), dict(y=None), dict(x=FAKE + 8), dict(y=FAKE), dict(given=4),
                dict(given=0),                                   # a statistics pass needs the workspace
                dict(sc=_layer(), given=G | SG),                 # a shortcut BN needs the residual
                dict(r=FAKE + 8192, sc=_layer(), given=G)]:      # the shortcut's statistics pass needs it too
        assert call(**bad) == -1, bad
        assert b"moco_bn_fwd_train_given" in lib.moco_last_error()
    assert call(given=0, work=FAKE, nbytes=ws - 1) == -3
    assert call(C=96) == -2                                      # C not a power of two
    assert _lib.launches == before
