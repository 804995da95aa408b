"""Argument validation of the frozen-BatchNorm entry points moco_bn_eval_act, moco_bn_relu_maxpool_eval and
moco_bn_eval_act_avgpool (include/moco_b200.h).  Every call here is refused before any kernel is launched, so no GPU
is needed."""
from moco_b200 import _lib

FAKE = 1 << 20                      # a 16-byte aligned address that is never dereferenced: validation fails first
S, T, S2, T2 = FAKE + 1 * 65536, FAKE + 2 * 65536, FAKE + 3 * 65536, FAKE + 4 * 65536


def _act(lib, x=FAKE, res=None, y=FAKE + 4096, M=1000, C=64, s=S, t=T, relu=1, s2=None, t2=None):
    return lib.moco_bn_eval_act(x, res, y, M, C, s, t, relu, s2, t2, None)


def _pool(lib, x=FAKE, res=None, feat=FAKE + 4096, N=3, HW=49, C=64, s=S, t=T, relu=1, s2=None, t2=None):
    return lib.moco_bn_eval_act_avgpool(x, res, feat, N, HW, C, s, t, relu, s2, t2, None)


def _stem(lib, x=FAKE, y=FAKE + 4096, N=2, H=9, W=9, C=64, s=S, t=T):
    return lib.moco_bn_relu_maxpool_eval(x, y, N, H, W, C, s, t, None)


def test_bn_eval_act_validates_its_arguments():
    lib = _lib.load()
    for rc in (_act(lib, x=None), _act(lib, y=None), _act(lib, s=None), _act(lib, t=None),
               _act(lib, x=FAKE + 8), _act(lib, y=FAKE + 4100), _act(lib, res=FAKE + 8200, s2=S2, t2=T2),
               _act(lib, res=FAKE + 8), _act(lib, y=FAKE), _act(lib, res=FAKE + 4096),
               _act(lib, res=FAKE + 8192, s2=S2), _act(lib, res=FAKE + 8192, t2=T2),
               _act(lib, s2=S2, t2=T2)):                       # a shortcut BN without a residual
        assert rc == -1
    assert _act(lib, res=FAKE + 8192, s2=S2) == -1 and b"moco_bn_eval_act" in lib.moco_last_error()
    assert _act(lib, C=96) == -2 and b"power of two" in lib.moco_last_error()
    assert _act(lib, C=4096) == -2
    assert _act(lib, C=32) == -2
    assert _act(lib, M=0) == -2


def test_bn_eval_act_avgpool_validates_its_arguments():
    lib = _lib.load()
    for rc in (_pool(lib, x=None), _pool(lib, feat=None), _pool(lib, s=None), _pool(lib, t=None),
               _pool(lib, x=FAKE + 8), _pool(lib, feat=FAKE + 4100), _pool(lib, res=FAKE + 8),
               _pool(lib, res=FAKE + 8192, s2=S2), _pool(lib, res=FAKE + 8192, t2=T2), _pool(lib, s2=S2, t2=T2)):
        assert rc == -1 and b"moco_bn_eval_act_avgpool" in lib.moco_last_error()
    assert _pool(lib, C=96) == -2 and b"power of two" in lib.moco_last_error()
    assert _pool(lib, C=4096) == -2
    assert _pool(lib, N=0) == -2 and _pool(lib, HW=0) == -2


def test_bn_relu_maxpool_eval_validates_its_arguments():
    lib = _lib.load()
    for rc in (_stem(lib, x=None), _stem(lib, y=None), _stem(lib, s=None), _stem(lib, t=None), _stem(lib, x=FAKE + 8),
               _stem(lib, y=FAKE + 4), _stem(lib, y=FAKE)):
        assert rc == -1 and b"moco_bn_relu_maxpool_eval" in lib.moco_last_error()
    assert _stem(lib, C=96) == -2 and b"power of two" in lib.moco_last_error()
    assert _stem(lib, C=4096) == -2
    assert _stem(lib, N=0) == -2 and _stem(lib, H=0) == -2 and _stem(lib, W=0) == -2


def test_eval_entry_points_are_counted_as_one_launch_each():
    assert all(_lib._Counting._PER_CALL[n] == 1
               for n in ("moco_bn_eval_act", "moco_bn_relu_maxpool_eval", "moco_bn_eval_act_avgpool"))
