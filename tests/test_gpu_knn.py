"""moco_knn and the kNN evaluation on the GPU (include/moco_b200.h: moco_knn; moco_b200/knn.py).

The features lie on a grid (multiples of 1/4 in [-1/2, 1/2]) where every bf16 dot product and every partial sum of it
is exact in fp32, so the similarities have one value whatever the summation order and the neighbour indices must equal
the oracle's exactly: the float64 numpy oracle (oracle/knn_oracle.py) on small cases, and ``reference_knn`` (exact
fp32 similarities from the same grid, a stable sort in the contract's order) on large ones.  The grid makes ties in s
common, so the (s descending, j ascending) order is exercised everywhere.  Scores are within SCORE_RTOL(k) of the
oracle's: expf is within 2 ulp and each class adds at most k positive terms in fp32.
"""
import gc
import importlib.util
import os

import numpy as np
import pytest
import torch

from moco_b200 import _lib
from moco_b200.knn import knn_predict, reference_knn
from oracle import knn_oracle as KO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 0.07


def SCORE_RTOL(k):
    return (k + 4) * 2.0 ** -23


@pytest.fixture(scope="module", autouse=True)
def _release():
    """Hand back to the driver the device memory of the large banks and their reference sorts, and the pinned host
    memory of the program's loader (pin_memory=True), both left in torch's caches, so that the tests after this module
    in the same process run with the memory they would have had without it."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch._C._host_emptyCache()


def _grid(g, n, c, lo=-2, hi=2):
    return (torch.randint(lo, hi + 1, (n, c), generator=g, device="cuda") * 0.25).bfloat16()


def _case(seed, nq, nb, c, n_classes=100):
    g = torch.Generator(device="cuda").manual_seed(seed)
    bank, q = _grid(g, nb, c), _grid(g, nq, c)
    labels = torch.randint(0, n_classes, (nb,), generator=g, device="cuda", dtype=torch.int32)
    return bank, labels, q


def _check_against(r, o_idx, o_sims, o_top, o_pred, o_scores, k):
    assert np.array_equal(r.indices.cpu().numpy(), o_idx)
    assert np.array_equal(r.sims.cpu().numpy(), np.asarray(o_sims, np.float32))
    np.testing.assert_allclose(r.scores.cpu().numpy(), o_top, rtol=SCORE_RTOL(k), atol=2.0 ** -126)
    ok = ~KO.ambiguous(o_scores, SCORE_RTOL(k))
    assert ok.any() or len(ok) < 8                              # some predictions are compared
    assert np.array_equal(r.pred.cpu().numpy()[ok], o_pred[ok])


# (C, Nq, Nb, k): C in {64, 128, 192, 2048}; Nq at 1, 63, 64, 65, 256, 1024; Nb at k, around the 128-row tile and the
# 1024-row slice group and their multiples; k in {1, 200, 1024}
SMALL = [(64, 1, 200, 200), (64, 63, 127, 1), (128, 64, 128, 1), (128, 65, 129, 129), (192, 1, 1023, 200),
         (192, 64, 1024, 1024), (64, 65, 1025, 1024), (128, 256, 3071, 200), (2048, 63, 3073, 200),
         (2048, 256, 2048, 1), (128, 1024, 4097, 1024), (192, 1024, 9000, 200)]


@pytest.mark.parametrize("c,nq,nb,k", SMALL)
def test_exact_against_the_float64_oracle(c, nq, nb, k):
    bank, labels, q = _case(c * 7 + nq + nb + k, nq, nb, c)
    r = knn_predict(bank, labels, q, k, T, 100, return_neighbors=True)
    o = KO.knn(q.float().cpu().numpy(), bank.float().cpu().numpy(), labels.cpu().numpy(), k, T, 100)
    _check_against(r, o["idx"], o["sims"], o["top"], o["pred"], o["scores"], k)


def _scores_np(ref, n_classes, labels):
    """float64 class scores of reference_knn's neighbours, for the ambiguity test."""
    idx, sims = ref.indices.cpu().numpy(), ref.sims.cpu().numpy().astype(np.float64)
    lab = labels.cpu().numpy()[idx]
    w = np.exp((sims - sims[:, :1]) / T)
    sc = np.zeros((idx.shape[0], n_classes))
    np.add.at(sc, (np.arange(idx.shape[0])[:, None].repeat(idx.shape[1], 1), lab), w)
    return sc


def _against_reference(bank, labels, q, k, n_classes=100, chunk=64):
    """reference_knn on `chunk` queries at a time: its [chunk, Nb] similarities and their sort stay a few GB even at
    ImageNet's bank size, so this module leaves the device as uncrowded as the rest of the suite does."""
    r = knn_predict(bank, labels, q, k, T, n_classes, return_neighbors=True)
    parts = [reference_knn(bank, labels, q[s:s + chunk], k, T, n_classes) for s in range(0, q.shape[0], chunk)]
    ref = type(parts[0])(*[None if p[0] is None else torch.cat(list(p)) for p in zip(*parts)])
    sc = _scores_np(ref, n_classes, labels)
    top = -np.sort(-sc, axis=1)[:, :5]
    pred = np.stack([np.lexsort((np.arange(n_classes), -row))[:5] for row in sc])
    _check_against(r, ref.indices.cpu().numpy(), ref.sims.cpu().numpy(), top, pred, sc, k)
    return r


@pytest.mark.parametrize("c,nq,k", [(128, 256, 200), (64, 1024, 1024), (2048, 65, 1)])
def test_exact_at_imagenet_bank_size(c, nq, k):
    bank, labels, q = _case(11 + c, nq, 1_281_167, c, 1000)
    _against_reference(bank, labels, q, k, 1000)


def test_exact_past_four_gigabytes_of_bank():
    nb, c = 1_100_000, 2048                                      # 4.5 GB: row offsets past 2^32 bytes
    assert nb * c * 2 > 2 ** 32
    bank, labels, q = _case(5, 64, nb, c, 1000)
    q[7] = bank[nb - 3]                                          # a neighbour past 2^32 bytes
    r = _against_reference(bank, labels, q, 200, 1000)
    assert (r.indices[7] == nb - 3).any()


def test_planted_ties_across_tile_group_and_cta_boundaries():
    """Copies of each query at rows that straddle the 128-row tiles, the 1024-row slice groups and the CTAs' 3072-row
    ranges (one query slice on a 132-SM H100: 293 groups, 3 per CTA), shifted by 12288 rows from query to query: the
    copies tie for the top, and the k = 4 first are the ones with the smallest j."""
    nb, c, nq = 300_000, 128, 16
    g = torch.Generator(device="cuda").manual_seed(3)
    bank = _grid(g, nb, c, -1, 1)
    labels = torch.randint(0, 10, (nb,), generator=g, device="cuda", dtype=torch.int32)
    q = _grid(g, nq, c, -1, 1)
    base = [127, 128, 1023, 1024, 2047, 2048, 3071, 3072, 6143, 6144]
    planted = []
    for i in range(nq):
        rows = [12288 * i + r for r in base[i % 5:]] + ([nb - 1] if i == 0 else [])
        bank[torch.tensor(rows, device="cuda")] = q[i]
        planted.append(sorted(rows)[:4])
    r = _against_reference(bank, labels, q, 4, 10)
    assert r.indices.tolist() == planted


def test_deterministic_across_runs_and_capacities():
    bank, labels, q = _case(21, 300, 200_000, 128, 50)
    y = torch.randint(0, 50, (300,), device="cuda")
    runs = [knn_predict(bank, labels, q, 200, T, 50, targets=y, return_neighbors=True, capacity=cap)
            for cap in (None, None, 200, 1 << 17)]
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)


def test_capacity_overflow_reruns_with_what_it_needs():
    """Identical bank rows: every row ties with every other, so each query's candidates are the whole bank."""
    nb, k = 5000, 200
    g = torch.Generator(device="cuda").manual_seed(4)
    row = _grid(g, 1, 64)
    bank = row.expand(nb, 64).contiguous()
    labels = torch.randint(0, 7, (nb,), generator=g, device="cuda", dtype=torch.int32)
    q = _grid(g, 33, 64)
    lib = _lib.load()
    import ctypes
    nbytes = lib.moco_knn_workspace_bytes(33, nb, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    top5 = torch.empty(33, 5, dtype=torch.int32, device="cuda")
    need = ctypes.c_int64(0)
    rc = lib.moco_knn(q.data_ptr(), bank.data_ptr(), labels.data_ptr(), 33, nb, 64, k, 1 / T, 7, None,
                      top5.data_ptr(), None, None, None, None, ws.data_ptr(), nbytes, ctypes.byref(need),
                      _lib.cur_stream())
    assert rc == _lib.ERR_CAPACITY and need.value == nb
    assert b"candidates" in lib.moco_last_error()
    before = _lib.launches
    r = knn_predict(bank, labels, q, k, T, 7, return_neighbors=True, capacity=k)
    assert _lib.launches - before == 8                           # four launches, then four again with the room
    o = KO.knn(q.float().cpu().numpy(), bank.float().cpu().numpy(), labels.cpu().numpy(), k, T, 7)
    assert (o["idx"] == np.arange(k)).all()
    _check_against(r, o["idx"], o["sims"], o["top"], o["pred"], o["scores"], k)


def test_launch_count_and_correct_counts():
    bank, labels, q = _case(8, 1500, 20_000, 128, 10)
    y = torch.randint(0, 10, (1500,), device="cuda")
    knn_predict(bank, labels, q[:8], 50, T, 10)                 # warm-up: set the kernels' smem attributes
    before = _lib.launches
    r = knn_predict(bank, labels, q, 50, T, 10, targets=y)
    assert _lib.launches - before == 8                           # two chunks (1024 + 476 queries), four launches each
    pred = r.pred
    assert int(r.correct[0]) == int((pred[:, 0] == y).sum())
    assert int(r.correct[1]) == int((pred == y[:, None]).any(1).sum())


def test_label_outside_the_classes_is_refused():
    bank, labels, q = _case(9, 4, 1000, 64, 10)
    labels[:] = 12
    with pytest.raises(RuntimeError, match="label"):
        knn_predict(bank, labels, q, 10, T, 10)


# ---- the whole program ---------------------------------------------------------------------------------------------
def _program():
    spec = importlib.util.spec_from_file_location("eval_knn_gpu", os.path.join(ROOT, "examples", "eval_knn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _split(root, split, n, seed0):
    import torchvision
    g = torch.Generator().manual_seed(seed0)
    for c in range(3):
        os.makedirs(os.path.join(root, split, f"c{c}"), exist_ok=True)
    for i in range(n):
        h = int(torch.randint(60, 300, (1,), generator=g))
        w = int(torch.randint(60, 300, (1,), generator=g))
        yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        img = torch.stack([(yy * 255) // h, (xx * 255) // w, ((yy + xx) * (3 + i % 3)) % 256]) + torch.randint(
            0, 40, (3, h, w), generator=g)
        data = torchvision.io.encode_jpeg(img.clamp(0, 255).to(torch.uint8).contiguous(), quality=90)
        with open(os.path.join(root, split, f"c{i % 3}", f"{i}.jpg"), "wb") as f:
            f.write(data.numpy().tobytes())


@pytest.mark.parametrize("layer", [7, 6])
def test_program_matches_reference_knn_on_its_bank(tmp_path, layer):
    from torch.utils.data import DataLoader
    from moco_b200 import augment as A
    from moco_b200.encoders import resnet50
    from moco_b200.knn import build_bank
    from moco_b200.linear_eval import ShardSampler
    root = str(tmp_path / "jpegs")
    _split(root, "train", 23, 0)
    _split(root, "val", 11, 100)
    torch.manual_seed(0)
    model = resnet50().cuda().to(memory_format=torch.channels_last)
    ckpt = str(tmp_path / "ckpt.pth")
    torch.save({"model": model.state_dict(), "epoch": 3}, ckpt)
    k = 5
    res = _program().main(["--data-dir", root, "--pretrained-model", ckpt, "--layer", str(layer), "--knn-k", str(k),
                           "--total-batch-size", "4", "--num-workers", "0"])
    assert res["n"] == 11 and res["bank"] == (23, 128 if layer == 7 else 2048)

    model.freeze()
    ds = A.ImageFolderEval(os.path.join(root, "train"), train=False)
    serial = DataLoader(ds, batch_size=4, shuffle=False, collate_fn=ds.collate_fn)
    sharded = DataLoader(ds, batch_size=4, sampler=ShardSampler(len(ds), 0, 1), collate_fn=ds.collate_fn)
    bank, labels = build_bank(model, sharded, layer)
    bank_s, labels_s = build_bank(model, serial, layer)
    assert torch.equal(bank, bank_s) and torch.equal(labels, labels_s)
    assert labels.tolist() == [ds.targets[i] for i in range(len(ds))]

    vds = A.ImageFolderEval(os.path.join(root, "val"), train=False)
    hits = np.zeros(2)
    for b in DataLoader(vds, batch_size=4, collate_fn=vds.collate_fn):
        x = A.resize_center_crops(b, dtype=torch.bfloat16, device="cuda")
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            f = model(x, layer).float()
        if layer == 6:
            f = f / f.pow(2).sum(1, keepdim=True).sqrt()
        y = b[2].cuda()
        ref = reference_knn(bank, labels, f, k, T, 3)
        hits += [(ref.pred[:, 0] == y).sum().item(), (ref.pred == y[:, None]).any(1).sum().item()]
    assert res["acc"] == pytest.approx(list(100.0 * hits / 11), abs=1e-9)
