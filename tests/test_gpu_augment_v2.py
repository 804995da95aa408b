"""MoCo v2 on the GPU: moco_augment_crops_blur against its exact restatement (tests/augment_blur_oracle.py) bit for bit
over tests/augment_blur_cases.py, an image past byte 2^32 and a 65535-crop batch, with three launches per call and
bit-identical reruns; a seeded V2 batch from a JPEG folder against torchvision's tensor transform within the derived
bound; MoCoStep with the MLP head against an eager statement of the step and with the fused tail; and the recipe with
--aug V2 --mlp, resumed bit-identically, its checkpoint scored by both eval examples."""
import ctypes
import itertools
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from moco_b200 import _lib, checkpoint
from moco_b200 import augment as MA
from tests import augment_blur_cases as BC
from tests.test_gpu_augment_exact import BIG_OFFSET, _assert_exact, _check_means, _pack
from tests.test_gpu_pretrain import _assert_same, _module, _recipe, folder  # noqa: F401  (the JPEG folder fixture)
from tests.test_host_augment_v2 import _bounds

pytestmark = pytest.mark.gpu
CASES = {c.name: c for c in BC.cases()}


def _augment(pix, recs, out, ksize, dtype=torch.float32):
    oh, ow = out
    prm = torch.from_numpy(np.ascontiguousarray(recs)).cuda()
    n = prm.shape[0]
    dst = torch.empty(n, 3, oh, ow, dtype=dtype, device="cuda")
    means = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    before = _lib.launches
    _lib.check(_lib.load().moco_augment_crops_blur(pix.data_ptr(), pix.numel(), prm.data_ptr(), n, oh, ow, ksize,
                                                   (ctypes.c_float * 6)(*BC.NORM), dst.data_ptr(),
                                                   _lib.dtype_code(dst), means.data_ptr(), _lib.cur_stream()),
               "moco_augment_crops_blur")
    torch.cuda.synchronize()
    assert _lib.launches - before == 3
    return dst.cpu(), means.cpu().numpy()


def _check(name, pix, recs, out, ksize, want, want_means):
    got, means = _augment(pix, recs, out, ksize)
    _assert_exact(name, got, want)
    _check_means(name, recs, means, want_means)
    again, _ = _augment(pix, recs, out, ksize)
    assert torch.equal(again, got), name
    bf, _ = _augment(pix, recs, out, ksize, torch.bfloat16)
    assert torch.equal(bf, got.to(torch.bfloat16)), name


@pytest.mark.parametrize("name", list(CASES))
def test_blur_case(name):
    case = CASES[name]
    img = case.image()
    pix, (off,) = _pack([img])
    want, want_means = BC.oracle(case, img)
    _check(name, pix, BC.records(case, off), case.out, case.ksize, want, want_means)


def test_image_past_byte_2_to_the_32():
    case = CASES["224/k23"]
    img = case.image()
    pix = torch.empty(BIG_OFFSET + img.nbytes, dtype=torch.uint8, device="cuda")
    pix[BIG_OFFSET:] = torch.from_numpy(img.reshape(-1)).cuda()
    want, want_means = BC.oracle(case, img)
    _check("past 2^32", pix, BC.records(case, BIG_OFFSET), case.out, case.ksize, want, want_means)
    del pix
    torch.cuda.empty_cache()


def test_65535_crops():
    """The grid limit: 65535 16 x 16 crops (ksize 31) over 3 images, 2 boxes and the 7 variants."""
    n, out, ksize = 65535, (16, 16), 31
    images = [BC.AC.image(40, 50, seed=700 + k) for k in range(3)]
    boxes = [(0, 0, 40, 50), (10, 5, 17, 30)]
    pix, offs = _pack(images)
    groups = list(itertools.product(range(3), range(2), range(len(BC.VARIANTS))))
    g_of = np.arange(n) % len(groups)
    recs = np.zeros((n, MA.V2_WORDS), np.int32)
    want = np.zeros((n, 3) + out, np.float32)
    want_means = np.zeros(n, np.float32)
    for gi, (a, b, v) in enumerate(groups):
        case = BC.BlurCase("g", out, (40, 50, 700 + a), ksize, [tuple(boxes[b]) + tuple(BC.VARIANTS[v])])
        sel = np.flatnonzero(g_of == gi)
        recs[sel] = BC.records(case, offs[a])
        o, m = BC.oracle(case, images[a])
        want[sel], want_means[sel] = o[0], m[0]
    _check("65535 crops", pix, recs, out, ksize, want, want_means)


def test_seeded_v2_batch_from_jpegs_is_torchvisions_within_the_bound(folder):  # noqa: F811
    ds = MA.ImageFolderTwoCrop(os.path.join(folder, "train"), scale=(0.2, 1.0), aug="V2")
    torch.manual_seed(21)
    items = [ds[i] for i in range(len(ds))]
    pixels, params, _ = MA.ImageFolderTwoCrop.collate_fn(items)
    assert params.shape[1] == MA.V2_WORDS and int(params[:, MA.BLUR].sum()) > 0
    out = MA.augment_crops((pixels, params), 224, dtype=torch.float32).cpu()
    worst = 0.0
    for k in range(params.shape[0]):
        r = params[k].tolist()
        img = items[k // 2][0]
        ref = MA.reference_crop(img, params[k]).numpy()
        f = params[k, MA.BRIGHTNESS:MA.WORDS].clone().view(torch.float32).tolist()
        # the bound reads the blur's weights only through their sum, 1 to a few ulps for every sigma: take sigma 2
        case = BC.BlurCase("jpeg", (224, 224), (r[MA.SRC_H], r[MA.SRC_W], 0), MA.BLUR_KSIZE,
                           [(r[MA.TOP], r[MA.LEFT], r[MA.HEIGHT], r[MA.WIDTH], r[MA.FLAGS], r[MA.ORDER], *f,
                             r[MA.GRAY_LATE], r[MA.BLUR], 2.0)])
        bound = float((_bounds(case) + _bounds(case, two_d=True))[0])
        err = float(np.abs(out[k].numpy() - ref).max())
        assert err <= bound, (k, err, bound)
        worst = max(worst, err / bound)
    print(f"largest |kernel - torchvision| / bound = {worst:.3g}")


# ------------------------------------------------------------------------------------------------ the MLP head

def _mlp_models(seed=0):
    from moco_b200 import encoders
    torch.manual_seed(seed)
    model = encoders.resnet18(low_dim=128, mlp=True).cuda()
    ema = encoders.resnet18(low_dim=128, mlp=True).cuda()
    ema.load_state_dict(model.state_dict())
    return model, ema


def test_mlp_step_matches_an_eager_statement():
    """One fp32 MoCoStep with the MLP head against the same step written in eager PyTorch: the two encoders
    (ShuffleBN on one GPU permutes the key batch, which batch statistics do not see), normalisation, the logits
    against the queue, cross-entropy on the positive, and the query encoder's gradients."""
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        N, K, T = 16, 256, 0.2
        model, ema = _mlp_models()
        twin, twin_ema = _mlp_models()
        contrast = MemoryMoCo(128, K, T).cuda()
        queue = contrast.memory.clone().bfloat16().float()
        contrast.memory.copy_(queue)
        opt = torch.optim.SGD(model.parameters(), lr=0.0, momentum=0.9)
        step = MoCoStep(model, ema, contrast, opt, alpha=0.999, amp_dtype=None)
        g = torch.Generator(device="cuda").manual_seed(3)
        batch = torch.randn(N, 6, 64, 64, device="cuda", generator=g)
        x1, x2 = torch.split(batch, [3, 3], dim=1)
        loss, _ = step(x1.contiguous(), x2.contiguous(), 1)

        twin.train()
        twin_ema.train()
        q = F.normalize(twin.fc(twin(x1.contiguous(), 6)), dim=1)
        with torch.no_grad():
            k = F.normalize(twin_ema.fc(twin_ema(x2.contiguous(), 6)), dim=1)
        logits = torch.cat([(q * k).sum(1, keepdim=True), q @ queue.t()], 1) / T
        ref = F.cross_entropy(logits, torch.zeros(N, dtype=torch.long, device="cuda"))
        ref.backward()
        assert abs(float(loss) - float(ref)) < 1e-2 * max(1.0, float(ref)), (float(loss), float(ref))
        for (name, p), p2 in zip(model.named_parameters(), twin.parameters()):
            if name.startswith("fc."):
                rel = float((p.grad - p2.grad).norm() / p2.grad.norm().clamp_min(1e-12))
                assert rel < 5e-2, (name, rel)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("graph", [False, True])
def test_mlp_step_with_fused_normalize_and_graphed_tail_matches_plain_step(graph):
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep
    runs = []
    for fused in (False, True):
        model, ema = _mlp_models()
        contrast = MemoryMoCo(128, 80, 0.2, device_index=fused and graph).cuda()
        opt = torch.optim.SGD(model.parameters(), lr=1e-3, momentum=0.9, weight_decay=1e-4)
        step = MoCoStep(model, ema, contrast, opt, amp_dtype=None, fuse_normalize=fused, graph_tail=fused and graph)
        g = torch.Generator(device="cuda").manual_seed(4)
        out = []
        for it in range(5):
            batch = torch.randn(16, 6, 64, 64, device="cuda", generator=g)
            x1, x2 = torch.split(batch, [3, 3], dim=1)
            loss, prob = step(x1.contiguous(), x2.contiguous(), 1)
            out.append((float(loss), float(prob)))
        torch.cuda.synchronize()
        runs.append((out, contrast.memory.cpu().numpy().copy(), model.fc[2].weight.detach().cpu().numpy().copy()))
    (o0, m0, w0), (o1, m1, w1) = runs
    for it, ((l0, p0), (l1, p1)) in enumerate(zip(o0, o1)):
        tol = 1e-2 if it < 3 else 3e-2
        assert abs(l0 - l1) < tol * max(1.0, abs(l0)), (it, o0, o1)
        assert abs(p0 - p1) < 5 * tol * max(p0, 1e-6) + 1e-6, (it, o0, o1)
    np.testing.assert_allclose(m0, m1, atol=5e-3)
    assert np.abs(w0 - w1).max() < 2e-2 * np.abs(w0).max()


def test_v2_mlp_recipe_resumes_bit_identically_and_evaluates(folder, tmp_path):  # noqa: F811
    mod = _module("train_moco_v2_gpu", "train_moco.py")
    flags = ["--aug", "V2", "--mlp", "--crop", "0.2", "--nce-t", "0.2", "--warmup-epoch", "0", "--persist-index"]
    a, b = str(tmp_path / "A"), str(tmp_path / "B")
    mod.main(_recipe(folder, a, *flags))
    mod.main(_recipe(folder, b, *flags, "--resume", os.path.join(a, "ckpt_epoch_1.pth")))
    ca, cb = checkpoint.load(os.path.join(a, "current.pth")), checkpoint.load(os.path.join(b, "current.pth"))
    assert ca["epoch"] == cb["epoch"] == 3 and ca["opt"]["aug"] == "V2" and ca["opt"]["mlp"] is True
    for key in ("model", "model_ema", "contrast", "optimizer", "scheduler"):
        _assert_same(ca[key], cb[key], key)
    assert "module.fc.0.weight" in ca["model"] and "module.fc.2.weight" in ca["model"]
    with pytest.raises(ValueError, match="MLP head"):
        mod.main(_recipe(folder, str(tmp_path / "C"), "--resume", os.path.join(a, "current.pth")))

    # the eval examples evaluate ResNet-50s: a one-epoch --mlp ResNet-50 run's checkpoint, at layers 7 and 6
    c = str(tmp_path / "R50")
    mod.main(_recipe(folder, c, *flags, arch="resnet50", epochs=1))
    path = os.path.join(c, "current.pth")
    knn = _module("eval_knn_v2_gpu", "eval_knn.py").main(
        ["--data-dir", folder, "--pretrained-model", path, "--layer", "7", "--knn-k", "5", "--num-workers", "0",
         "--total-batch-size", "8"])
    assert knn["bank"] == (24, 128) and knn["n"] == 7
    lin = _module("eval_linear_v2_gpu", "eval_linear.py").main(
        ["--pretrained", path, "--data-dir", folder, "--layer", "6", "--epochs", "1", "--total-batch-size", "4",
         "--num-workers", "0"])
    assert lin["n"] == 7 and np.isfinite(lin["loss"])
