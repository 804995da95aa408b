"""Argument validation of the sharded-queue entry points moco_nce_shard_merge, moco_nce_shard_dq_finish and
moco_nce_shard_dq_finish_peers (include/moco_b200.h).  Every call here has exactly one bad argument and is refused
before any kernel is launched, so no GPU is needed."""
import ctypes

from moco_b200 import _lib

FAKE = 1 << 20                      # a 256-byte aligned address that is never dereferenced: validation fails first
K_OWN, PROB, DQ, O_OWN = (FAKE + n * 65536 for n in range(1, 5))


def _peers(world, bad=None, value=None):
    ptrs = [FAKE + 8 * 65536 + r * 65536 for r in range(world)]
    if bad is not None:
        ptrs[bad] = value
    return (ctypes.c_void_p * world)(*ptrs)


def _merge(lib, world=2, N=8, C=128):
    return lib.moco_nce_shard_merge(FAKE, world, N, C, 14.0, FAKE + 4096, FAKE + 8192, FAKE + 12288, FAKE + 16384,
                                    FAKE + 65536, 1 << 24, None)


def _peers_call(lib, peers=None, world=4, rank=1, N=8, C=128):
    peers = _peers(world) if peers is None else peers
    return lib.moco_nce_shard_dq_finish_peers(peers, world, rank, K_OWN, _lib.MOCO_F32, PROB, N, C, 14.0, DQ, None)


def _finish(lib, o=O_OWN, k=K_OWN, prob=PROB, dq=DQ, N=8, C=128):
    return lib.moco_nce_shard_dq_finish(o, k, _lib.MOCO_F32, prob, N, C, 14.0, dq, None)


def test_shard_merge_rejects_world_out_of_range():
    lib = _lib.load()
    for world in (0, -1, 161):
        assert _merge(lib, world=world) == -1
        msg = lib.moco_last_error()
        assert b"moco_nce_shard_merge" in msg and b"world=%d" % world in msg


def test_shard_dq_finish_peers_validates_its_arguments():
    lib = _lib.load()
    cases = {
        "world 17": dict(peers=_peers(17), world=17, rank=0),
        "world 0": dict(peers=_peers(1), world=0, rank=0),
        "rank == world": dict(rank=4),
        "rank > world": dict(rank=9),
        "negative rank": dict(rank=-1),
        "null peer": dict(peers=_peers(4, bad=2, value=None)),
        "misaligned peer": dict(peers=_peers(4, bad=3, value=FAKE + 8 * 65536 + 8)),
        "C not a multiple of 4": dict(C=130),
        "N = 0": dict(N=0),
    }
    for what, kw in cases.items():
        assert _peers_call(lib, **kw) == -1, what
        assert b"moco_nce_shard_dq_finish_peers" in lib.moco_last_error(), what
    assert _peers_call(lib, peers=_peers(4, bad=2, value=None)) == -1 and b"peer 2" in lib.moco_last_error()
    assert lib.moco_nce_shard_dq_finish_peers(None, 4, 1, K_OWN, _lib.MOCO_F32, PROB, 8, 128, 14.0, DQ, None) == -1
    for null in ("k", "prob", "dq"):
        args = [K_OWN, PROB, DQ]
        args[("k", "prob", "dq").index(null)] = None
        assert lib.moco_nce_shard_dq_finish_peers(_peers(4), 4, 1, args[0], _lib.MOCO_F32, args[1], 8, 128, 14.0,
                                                  args[2], None) == -1, null


def test_shard_dq_finish_rejects_null_arguments():
    lib = _lib.load()
    for kw in (dict(o=None), dict(k=None), dict(prob=None), dict(dq=None), dict(N=0), dict(C=0)):
        assert _finish(lib, **kw) == -1, kw
        assert b"moco_nce_shard_dq_finish" in lib.moco_last_error(), kw

