"""Argument validation of moco_bn_add_relu_* and moco_bn_relu_maxpool_fwd_train (include/moco_b200.h), next to the
moco_bn_* checks of test_host_cpu.py.  Every call here is refused before any kernel is launched, so no GPU is needed."""
from moco_b200 import _lib

FAKE = 1 << 20                      # a 16-byte aligned address that is never dereferenced: validation fails first


def _layer(fwd=True, **kw):
    f = dict(gamma=FAKE, beta=FAKE, save_mean=FAKE, save_invstd=FAKE, momentum=0.1, eps=1e-5)
    if not fwd:
        f.update(dgamma=FAKE, dbeta=FAKE)
    f.update(kw)
    return _lib.BnLayer(**f)


def _fwd(lib, x=FAKE, res=FAKE, y=FAKE + 4096, mask=None, M=1024, C=64, bn=None, sc=None, ws=FAKE, wsb=None):
    wsb = lib.moco_bn_workspace_bytes() if wsb is None else wsb
    return lib.moco_bn_add_relu_fwd_train(x, res, y, mask, M, C, bn if bn is not None else _layer(), sc, ws, wsb, None)


def _bwd(lib, dy=FAKE, x=FAKE, res=None, mask=FAKE, M=1024, C=64, bn=None, sc=None, dx=FAKE, dres=None, ws=FAKE,
         wsb=None):
    wsb = lib.moco_bn_workspace_bytes() if wsb is None else wsb
    return lib.moco_bn_add_relu_bwd(dy, x, res, mask, M, C, bn if bn is not None else _layer(False), sc, dx, dres, ws,
                                    wsb, None)


def test_bn_add_relu_entry_points_validate_their_arguments():
    lib = _lib.load()
    # the workspace holds three per-channel sums per reduction CTA (the shortcut BN's backward)
    assert lib.moco_bn_workspace_bytes() >= 256 + 3 * 64 * 4
    for rc in (_fwd(lib, x=None), _fwd(lib, res=None), _fwd(lib, y=FAKE), _fwd(lib, res=FAKE + 4096),
               _fwd(lib, x=FAKE + 8), _fwd(lib, bn=_layer(eps=0.0)), _fwd(lib, bn=_layer(gamma=None)),
               _fwd(lib, bn=_layer(running_mean=FAKE)), _fwd(lib, sc=_layer(save_invstd=None))):
        assert rc == -1 and b"moco_bn_add_relu_fwd_train" in lib.moco_last_error()
    assert _fwd(lib, wsb=16) == -3
    assert _fwd(lib, C=96) == -2 and b"power of two" in lib.moco_last_error()
    assert _fwd(lib, C=4096) == -2
    assert _fwd(lib, M=0) == -2

    # the mask is required; a shortcut BN needs its input, its input gradient and dgamma / dbeta
    for rc in (_bwd(lib, mask=None), _bwd(lib, dy=None), _bwd(lib, dx=FAKE + 8),
               _bwd(lib, bn=_layer(False, dgamma=None)),
               _bwd(lib, sc=_layer(False), dres=FAKE + 4096),
               _bwd(lib, sc=_layer(False), res=FAKE + 8192),
               _bwd(lib, sc=_layer(False, dbeta=None), res=FAKE + 8192, dres=FAKE + 4096)):
        assert rc == -1 and b"moco_bn_add_relu_bwd" in lib.moco_last_error()
    assert _bwd(lib, wsb=0) == -3
    assert _bwd(lib, C=32) == -2 and b"power of two" in lib.moco_last_error()


def test_bn_relu_maxpool_entry_points_validate_their_arguments():
    lib = _lib.load()
    wsb = lib.moco_bn_workspace_bytes()

    def fwd(x=FAKE, y=FAKE + 4096, taps=FAKE + 8192, N=2, H=9, W=9, C=64, bn=None, wsb=wsb):
        return lib.moco_bn_relu_maxpool_fwd_train(x, y, taps, N, H, W, C, bn if bn is not None else _layer(), FAKE,
                                                  wsb, None)

    for rc in (fwd(x=None), fwd(taps=None), fwd(taps=FAKE + 4), fwd(y=FAKE + 8), fwd(bn=_layer(eps=-1.0))):
        assert rc == -1 and b"moco_bn_relu_maxpool_fwd_train" in lib.moco_last_error()
    assert fwd(wsb=8) == -3
    assert fwd(C=72) == -2 and fwd(H=0) == -2
