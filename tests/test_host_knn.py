"""Host side of the weighted kNN evaluation, no GPU needed: the float64 oracle of the contract (include/moco_b200.h:
moco_knn) on hand-checked cases with planted ties, ``moco_b200.knn.reference_knn`` against it, every refusal of
moco_knn through the C ABI (before any launch) and examples/eval_knn.py's command line."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from moco_b200 import _lib
from moco_b200.knn import reference_knn
from oracle import knn_oracle as KO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rows(*vals):
    return np.array(vals, np.float64)


def test_oracle_breaks_similarity_ties_by_index():
    # s = 3, 2, 3, 1, 2 for rows 0..4: order (3, j=0), (3, j=2), (2, j=1), (2, j=4), (1, j=3)
    bank = _rows([3, 0], [2, 0], [3, 0], [1, 0], [2, 0])
    q = _rows([1, 0])
    r = KO.knn(q, bank, [0, 1, 2, 3, 4], k=3, t=1.0, n_classes=5)
    assert r["idx"].tolist() == [[0, 2, 1]]                 # the tie at the k-th place (rows 1 and 4) goes to j = 1
    assert r["sims"].tolist() == [[3, 3, 2]]
    # weights 1, 1, e^-1: classes 0 and 2 tie at 1, class 1 has e^-1; the rest 0, by class
    assert r["pred"].tolist() == [[0, 2, 1, 3, 4]]
    assert np.allclose(r["top"], [[1, 1, np.exp(-1), 0, 0]])


def test_oracle_breaks_class_score_ties_by_class():
    bank = _rows([1, 0], [1, 0], [1, 0], [1, 0])
    q = _rows([2, 0])
    r = KO.knn(q, bank, [3, 1, 3, 1], k=4, t=0.5, n_classes=6)
    assert r["idx"].tolist() == [[0, 1, 2, 3]]
    assert r["pred"].tolist() == [[1, 3, 0, 2, 4]]           # 1 and 3 score 2 each; then 0, 2, 4 at 0
    assert r["top"][0, :2].tolist() == [2.0, 2.0]


def test_oracle_at_nb_equal_k_and_k_1():
    bank = _rows([0, 1], [1, 0], [0.5, 0.5])
    q = _rows([1, 0], [0, 1])
    r = KO.knn(q, bank, [2, 0, 1], k=3, t=1.0, n_classes=3)   # Nb = k: every row, in order
    assert r["idx"].tolist() == [[1, 2, 0], [0, 2, 1]]
    assert r["pred"].tolist() == [[0, 1, 2, -1, -1], [2, 1, 0, -1, -1]]   # 3 classes: -1 past them
    r1 = KO.knn(q, bank, [2, 0, 1], k=1, t=1.0, n_classes=3)
    assert r1["idx"].tolist() == [[1], [0]]
    assert r1["pred"][:, 0].tolist() == [0, 2]
    assert r1["top"][:, 0].tolist() == [1.0, 1.0]              # exp(0)


def test_oracle_vote_weights_follow_the_temperature():
    bank = _rows([1.0, 0], [0.5, 0], [0.5, 0])
    q = _rows([1, 0])
    r = KO.knn(q, bank, [0, 1, 1], k=3, t=0.1, n_classes=2)
    assert np.isclose(r["scores"][0, 0], 1.0) and np.isclose(r["scores"][0, 1], 2 * np.exp(-5.0))
    assert r["pred"][0, :2].tolist() == [0, 1]
    r = KO.knn(q, bank, [0, 1, 1], k=3, t=1.0, n_classes=2)  # 2 e^-0.5 = 1.21 > 1
    assert r["pred"][0, :2].tolist() == [1, 0]


@pytest.mark.parametrize("seed,k,n_classes", [(0, 1, 3), (1, 7, 4), (2, 40, 10), (3, 64, 7)])
def test_reference_knn_matches_the_oracle(seed, k, n_classes):
    """Grid features (every dot product exact in fp32) with many ties in s."""
    g = np.random.default_rng(seed)
    nb, nq, c = 200, 9, 64
    bank = g.integers(-2, 3, (nb, c)) / 4.0
    bank[50:60] = bank[10]                                      # identical rows: ties at every rank they reach
    q = g.integers(-2, 3, (nq, c)) / 4.0
    q[3] = bank[10]
    labels = g.integers(0, n_classes, nb)
    o = KO.knn(q, bank, labels, k, 0.07, n_classes)
    r = reference_knn(torch.tensor(bank).bfloat16(), torch.tensor(labels, dtype=torch.int32),
                      torch.tensor(q).bfloat16(), k, 0.07, n_classes)
    assert np.array_equal(r.indices.numpy(), o["idx"])
    assert np.array_equal(r.sims.numpy(), o["sims"].astype(np.float32))
    np.testing.assert_allclose(r.scores.numpy(), o["top"][:, :5], rtol=1e-5, atol=0)
    ok = ~KO.ambiguous(o["scores"], 1e-5)
    assert ok.sum() >= nq // 2
    assert np.array_equal(r.pred.numpy()[ok], o["pred"][ok])


# ---- moco_knn's refusals (include/moco_b200.h) -------------------------------------------------------------------
FAKE = 0x10000                                                  # 256-byte aligned, never dereferenced
NQ, NB, C, K = 64, 4096, 128, 200


def _call(lib, q=FAKE, bank=FAKE + (1 << 20), labels=FAKE + (1 << 24), nq=NQ, nb=NB, c=C, k=K, inv_t=1 / 0.07,
          n_classes=10, targets=None, top5=FAKE + (1 << 26), scores=None, idx=None, sims=None, correct=None,
          ws=FAKE + (1 << 30), nbytes=None, need=True):
    if nbytes is None:
        nbytes = lib.moco_knn_workspace_bytes(max(nq, 1), max(nb, 1), max(k, 1)) or (1 << 24)
    out = ctypes.c_int64(0)
    return lib.moco_knn(q, bank, labels, nq, nb, c, k, inv_t, n_classes, targets, top5, scores, idx, sims, correct, ws,
                        nbytes, ctypes.byref(out) if need else None, None)


def test_knn_validates_its_arguments():
    lib = _lib.load()
    before = _lib.launches
    invalid = [dict(q=None), dict(bank=None), dict(labels=None), dict(top5=None), dict(ws=None), dict(need=False),
               dict(q=FAKE + 8), dict(bank=FAKE + (1 << 20) + 2), dict(ws=FAKE + (1 << 30) + 16),
               dict(labels=FAKE + (1 << 24) + 2), dict(top5=FAKE + (1 << 26) + 1),
               dict(targets=FAKE + (1 << 27)),                  # targets without correct
               dict(correct=FAKE + (1 << 27)),                  # and the reverse
               dict(inv_t=0.0), dict(inv_t=-1.0), dict(inv_t=float("inf")), dict(inv_t=float("nan")),
               dict(n_classes=0), dict(n_classes=65537), dict(k=0), dict(nb=K - 1)]
    for bad in invalid:
        assert _call(lib, **bad) == -1, bad
        assert b"moco_knn" in lib.moco_last_error()
    for bad in [dict(nq=0), dict(nq=1025), dict(c=0), dict(c=96), dict(c=2112), dict(c=32), dict(k=1025, nb=NB),
                dict(nb=1 << 31)]:
        assert _call(lib, **bad) == -2, bad
        assert b"moco_knn" in lib.moco_last_error()
    assert _lib.launches == before


def test_knn_refuses_overlapping_outputs():
    lib = _lib.load()
    before = _lib.launches
    top5 = FAKE + (1 << 26)
    t = FAKE + (1 << 27)
    for bad in [dict(top5=FAKE),                                 # over q
                dict(top5=FAKE + (1 << 20) + 4096),              # inside the bank
                dict(top5=FAKE + (1 << 24) + 64),                # inside the labels
                dict(top5=FAKE + (1 << 30) + 256),               # inside the workspace
                dict(scores=top5),                               # two outputs at one address
                dict(scores=top5 + 16),                          # overlapping by one element
                dict(idx=top5 + NQ * 20 - 4),
                dict(sims=FAKE + (1 << 28), idx=FAKE + (1 << 28) + NQ * K * 4 - 4),
                dict(targets=t, correct=t),                      # correct over the targets
                dict(targets=t, correct=top5 + 8)]:
        assert _call(lib, **bad) == -1, bad
        assert b"overlap" in lib.moco_last_error()
    assert _lib.launches == before


def test_knn_refuses_too_small_a_workspace():
    lib = _lib.load()
    need = lib.moco_knn_workspace_bytes(NQ, NB, K)                # room for k candidates per query
    assert need > 0 and lib.moco_knn_workspace_bytes(NQ, NB, K + 1) == need + NQ * 8
    assert _call(lib, nbytes=need - 1) == -3
    assert b"workspace too small" in lib.moco_last_error()
    for bad in [(0, NB, K), (1025, NB, K), (NQ, 0, 1), (NQ, NB, 0), (NQ, NB, NB + 1), (NQ, 1 << 31, K)]:
        assert lib.moco_knn_workspace_bytes(*bad) == 0, bad


# ---- examples/eval_knn.py's command line -------------------------------------------------------------------------
def _program():
    spec = importlib.util.spec_from_file_location("eval_knn_example", os.path.join(ROOT, "examples", "eval_knn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_eval_knn_defaults(monkeypatch):
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    a = _program().parse_args(["--data-dir", "D", "--pretrained-model", "P"])
    assert (a.data_dir, a.pretrained, a.layer, a.knn_k, a.knn_t, a.total_batch_size, a.num_workers, a.local_rank) == (
        "D", "P", 7, 200, 0.07, 256, 4, 0)


def test_eval_knn_flags():
    a = _program().parse_args(["--data-dir", "D", "--pretrained", "P", "--layer", "6", "--knn-k", "1024",
                               "--knn-t", "0.1", "--total-batch-size", "64", "--num-workers", "0"])
    assert (a.layer, a.knn_k, a.knn_t, a.total_batch_size, a.num_workers) == (6, 1024, 0.1, 64, 0)


@pytest.mark.parametrize("argv", [["--pretrained-model", "P"], ["--data-dir", "D"],     # each is required
                                  ["--layer", "5"], ["--knn-k", "0"], ["--knn-k", "1025"], ["--knn-t", "0"],
                                  ["--knn-t", "-1"], ["--total-batch-size", "0"]])
def test_eval_knn_rejects(argv):
    full = argv if len(argv) == 2 and argv[0] in ("--data-dir", "--pretrained-model") else \
        ["--data-dir", "D", "--pretrained-model", "P"] + argv
    with pytest.raises(SystemExit):
        _program().parse_args(full)


def test_eval_knn_launch_rank(monkeypatch):
    p = _program()
    base = ["--data-dir", "D", "--pretrained-model", "P"]
    monkeypatch.setenv("LOCAL_RANK", "3")
    assert p.parse_args(base).local_rank == 3
    assert p.parse_args(base + ["--local_rank", "1"]).local_rank == 1
    assert p.parse_args(base + ["--local-rank=2"]).local_rank == 2
    monkeypatch.delenv("LOCAL_RANK")
    assert p.parse_args(base).local_rank == 0
