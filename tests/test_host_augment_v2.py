"""MoCo v2 on the host, no GPU needed: the V2 sampler's draws against torchvision's Compose, the blur weights against
torchvision's, the oracle's blur and gray-after-jitter steps on the case table of tests/augment_blur_cases.py
(against torchvision and within a derived float64 bound, and each blur mutant caught), the 32-word validator and the C
entry's refusals, the example trainer's --aug V2 / --mlp, and MLP-head checkpoints.

The float64 bound extends test_host_augment_exact's (same units and notation) by the blur: one 1-D pass of n = 2h + 1
taps with float32 weights k (shared exactly by the float64 mode, S their float64 sum) over values in [0, A] that are
off by e gives S e + gamma_n S A; two passes, the second over values in [0, S A].  torchvision's conv2d sums the n^2
products of its rounded 2-D weights (each off by u relative) in its own order: S^2 e + (gamma_{n^2} + u) S^2 A.  Its
other stages are the same operations in another order, bounded by the same formulas, so |oracle - torchvision| is at
most the oracle's bound plus torchvision's.
"""
import argparse
import ctypes
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch
from torchvision.transforms import _functional_tensor as FT

from moco_b200 import _lib, checkpoint, encoders
from moco_b200 import augment as A
from oracle import augment_oracle as O
from tests import augment_blur_cases as BC
from tests import augment_blur_oracle as BO
from tests.test_host_augment_exact import U, A as VMAX, _gamma, _normalized, _pointwise_bound, _resample_bound, \
    _terms_per_thread

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def _image(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8)


# ------------------------------------------------------------------------------------------------ draws and weights

@pytest.mark.parametrize("hw", [(375, 500), (30, 600), (120, 150)])
def test_v2_sampler_and_reference_crop_equal_compose(hw):
    """40 seeds: sample_crop_params(aug="V2") + reference_crop == MoCo v2's Compose on the same RNG, bit for bit."""
    img = _image(*hw, seed=hw[1])
    x = img.permute(2, 0, 1).float() / 255
    comp = A.reference_compose("V2")
    seen = set()
    for seed in range(40):
        torch.manual_seed(seed)
        ref = comp(x)
        torch.manual_seed(seed)
        rec = A.sample_crop_params(*hw, aug="V2")
        assert rec.shape == (A.V2_WORDS,) and int(rec[A.GRAY_LATE]) == 1
        assert torch.equal(A.reference_crop(img, rec), ref), (hw, seed)
        seen.add((bool(rec[A.FLAGS] & _lib.AUG_JITTER), bool(rec[A.BLUR])))
    assert seen == {(False, False), (False, True), (True, False), (True, True)}


@pytest.mark.parametrize("ksize", [3, 23, 31])
@pytest.mark.parametrize("sigma", [0.1, 0.5, 1.7, 2.0])
def test_weights_are_torchvisions(ksize, sigma):
    k = FT._get_gaussian_kernel1d(ksize, sigma, torch.float32, torch.device("cpu"))
    half = A.gaussian_half_kernel(ksize, sigma)
    assert len(half) == 16 and half[:ksize // 2 + 1] == k[ksize // 2:].tolist() and not any(half[ksize // 2 + 1:])
    assert torch.equal(k, k.flip(0))
    assert np.array_equal(BC.kernel1d(ksize, sigma), k.numpy())


# ------------------------------------------------------------------------------------------------ the case table

def _blur_bound(e, k, two_d=False):
    n, S = len(k), float(np.sum(np.asarray(k, np.float64)))
    if two_d:
        return S * S * e + (_gamma(n * n) + U) * S * S * VMAX
    e1 = S * e + _gamma(n) * S * VMAX
    return S * e1 + _gamma(n) * S * S * VMAX


def _bounds(case, two_d=False):
    """Per crop: the float64 bound of the oracle (two_d=False) or of torchvision's evaluation (two_d=True)."""
    out_h, out_w = case.out
    res = []
    for top, left, ch, cw, flags, order, b, c, s, hue, late, blur, sigma in case.crops:
        ty, tx = O.Taps(np.arange(out_h), ch, out_h), O.Taps(np.arange(out_w), cw, out_w)
        L = _terms_per_thread(out_h, out_w, O.chunk_width(cw, out_w, out_w))
        e = _pointwise_bound(_resample_bound(ty, tx), flags, order, [b, c, s, hue], L)
        if late and flags & BC.GRAY:
            e += 3 * U * VMAX
        if blur:
            e = _blur_bound(e, BC.kernel1d(case.ksize, sigma), two_d)
        res.append(_normalized(e))
    return np.array(res)


@pytest.fixture(scope="module")
def table():
    rows = []
    for case in BC.cases():
        img = case.image()
        rows.append((case, img, BC.oracle(case, img), BC.oracle(case, img, exact=False)))
    return rows


def test_table_is_inside_the_contract():
    for case in BC.cases():
        A.validate_params_v2(torch.from_numpy(BC.records(case)), case.src[0] * case.src[1] * 3, case.out[1],
                             case.ksize)


def test_table_within_the_float64_bound(table):
    tightest = 0.0
    for case, img, got, ref in table:
        bound = _bounds(case)
        err = np.abs(got[0] - ref[0]).reshape(len(case.crops), -1).max(axis=1)
        assert (err <= bound).all(), (case.name, err, bound)
        tightest = max(tightest, float((err / bound).max()))
    print(f"largest error / bound = {tightest:.3g}")


def test_table_against_torchvision(table):
    worst = 0.0
    for case, img, got, _ in table:
        bound = _bounds(case) + _bounds(case, two_d=True)
        recs = BC.records(case)
        for k in range(len(case.crops)):
            tv = A.reference_crop(torch.from_numpy(img), torch.from_numpy(recs[k].copy()), case.out,
                                  ksize=case.ksize).numpy()
            err = float(np.abs(got[0][k] - tv).max())
            assert err <= bound[k], (case.name, k, err, bound[k])
            worst = max(worst, err / bound[k])
    print(f"largest |oracle - torchvision| / bound = {worst:.3g}")


def test_unblurred_v1_order_records_are_the_v1_oracle(table):
    """gray_after_jitter = blur = 0 is moco_augment_crops' computation."""
    for case, img, got, _ in table:
        for k, (top, left, ch, cw, flags, order, b, c, s, hue, late, blur, sigma) in enumerate(case.crops):
            if late or blur:
                continue
            o, _ = O.augment(img[top:top + ch, left:left + cw][None], *case.out, flags, order,
                             np.array([[b, c, s, hue]], np.float32), BC.NORM)
            assert np.array_equal(o[0], got[0][k]), case.name


@pytest.mark.parametrize("mutant", BO.BLUR_MUTANTS)
def test_blur_mutants_are_caught(table, mutant):
    differs = breaks = None
    for case, img, got, ref in table:
        mut = BC.oracle(case, img, mutant=mutant)
        over = (np.abs(mut[0] - ref[0]).reshape(len(case.crops), -1) > _bounds(case)[:, None]).any()
        differs = differs or (case.name if not np.array_equal(mut[0], got[0]) else None)
        breaks = breaks or (case.name if over else None)
        if differs and (breaks or mutant not in BO.BLUR_SEMANTIC_MUTANTS):
            break
    print(f"{mutant}: differs on {differs}, breaks the float64 bound on {breaks}")
    assert differs
    if mutant in BO.BLUR_SEMANTIC_MUTANTS:
        assert breaks


# ------------------------------------------------------------------------------------------------ validation

def _good():
    torch.manual_seed(1)
    recs = []
    while len(recs) < 4 or not any(int(r[A.BLUR]) for r in recs):
        recs.append(A.sample_crop_params(100, 120, aug="V2"))
    return torch.stack(recs), 100 * 120 * 3


def _f32(v):
    return int(torch.tensor([v], dtype=torch.float32).view(torch.int32))


@pytest.mark.parametrize("word,value,match", [
    (A.SRC_W, 121, "outside the pixel buffer"),
    (A.FLAGS, 8, "flag bits"),
    (A.GRAY_LATE, 2, "gray_after_jitter"),
    (A.BLUR, -1, "blur is not"),
    (A.WEIGHTS, _f32(float("nan")), "non-finite"),
    (A.WEIGHTS + 3, _f32(-0.01), "outside"),
    (A.WEIGHTS + 5, _f32(1.5), "outside"),
    (A.WEIGHTS + 12, _f32(0.001), "past ksize"),
])
def test_malformed_v2_records_raise_value_error(word, value, match):
    params, nbytes = _good()
    A.validate_params_v2(params, nbytes, 224)
    bad = params.clone()
    bad[1, word] = value
    with pytest.raises(ValueError, match=match):
        A.validate_params_v2(bad, nbytes, 224)


def test_v2_validator_refuses_shapes_and_ksize():
    params, nbytes = _good()
    with pytest.raises(ValueError, match=r"\[n, 32\]"):
        A.validate_params_v2(params[:, :A.WORDS], nbytes)
    with pytest.raises(ValueError, match="ksize"):
        A.validate_params_v2(params, nbytes, ksize=22)
    with pytest.raises(ValueError, match="past ksize"):
        A.validate_params_v2(params, nbytes, ksize=3)


def test_blur_entry_validates_its_arguments_without_a_gpu():
    lib = _lib.load()
    norm = (ctypes.c_float * 6)(*A.MEAN, *A.STD)
    addr = 0x7f0000001000
    args = [addr, 1000, addr + 0x1000, 2, 224, 224, 23, norm, addr + 0x2000, _lib.MOCO_BF16, addr + 0x3000, None]
    for k, v in ((0, None), (1, 0), (2, addr + 4), (9, 7), (10, addr + 2), (4, 0), (5, 513), (4, 513), (3, 70000),
                 (6, 22), (6, 1), (6, 33), (6, 0)):
        a = list(args)
        a[k] = v
        assert lib.moco_augment_crops_blur(*a) == -1, (k, v)
        assert b"moco_augment_crops_blur" in lib.moco_last_error()
    for oh, ow, ks in ((16, 16, 33), (15, 200, 31), (200, 11, 23), (1, 1, 3)):      # ksize // 2 < min(out_h, out_w)
        a = list(args)
        a[4:7] = [oh, ow, ks]
        assert lib.moco_augment_crops_blur(*a) == -1 and b"ksize" in lib.moco_last_error(), (oh, ow, ks)
    a = list(args)
    a[7] = (ctypes.c_float * 6)(*A.MEAN, 0.2, 0.0, 0.2)
    assert lib.moco_augment_crops_blur(*a) == -1 and b"std" in lib.moco_last_error()
    a = list(args)
    a[3] = 0
    assert lib.moco_augment_crops_blur(*a) == 0          # no crops: nothing is launched


def test_header_declares_the_blur_record_and_launch_count():
    text = open(os.path.join(ROOT, "include", "moco_b200.h")).read()
    assert "} moco_aug_crop_blur;                     /* 128 bytes" in text
    assert "Three launches" in text and "int moco_augment_crops_blur(" in text


# ------------------------------------------------------------------------------------------------ the recipe

def _trainer(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "examples", "train_moco.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_trainer_parses_aug_v2_and_mlp():
    mod = _trainer("train_moco_v2_flags")
    a = mod.parse_args(["--data-dir", "/d"])
    assert (a.aug, a.mlp, a.crop, a.nce_t, a.base_lr, a.batch_size, a.warmup_epoch) == ("CJ", False, 0.08, 0.07, 0.1,
                                                                                         128, 5)
    a = mod.parse_args(["--data-dir", "/d", "--aug", "V2", "--mlp", "--crop", "0.2", "--nce-t", "0.2", "--base-lr",
                        "0.03", "--batch-size", "256", "--lr-scheduler", "cosine", "--warmup-epoch", "0"])
    assert (a.aug, a.mlp, a.crop, a.nce_t, a.base_lr, a.batch_size, a.warmup_epoch) == ("V2", True, 0.2, 0.2, 0.03,
                                                                                         256, 0)


def test_v2_loader_yields_32_word_records(tmp_path):
    from tests.test_host_augment import _jpeg_folder
    mod = _trainer("train_moco_v2_loader")
    _jpeg_folder(str(tmp_path), [(40, 48)] * 4)
    args = mod.parse_args(["--data-dir", str(tmp_path), "--batch-size", "2", "--num-workers", "0", "--aug", "V2"])
    pixels, params, _ = next(iter(mod.make_loader(args, world=1)))
    assert params.shape == (4, A.V2_WORDS)
    A.validate_params_v2(params, pixels.numel(), 224)


def _mlp_state(arch="resnet18"):
    torch.manual_seed(0)
    ctor = getattr(encoders, arch)
    model, ema = ctor(mlp=True), ctor(mlp=True)
    return model, ema


def test_mlp_head_layout_and_default():
    model = encoders.resnet50(mlp=True)
    keys = [k for k in model.state_dict() if k.startswith("fc.")]
    assert keys == ["fc.0.weight", "fc.0.bias", "fc.2.weight", "fc.2.bias"]
    assert model.fc[0].weight.shape == (2048, 2048) and model.fc[2].weight.shape == (128, 2048)
    assert (model.feat_dim, model.low_dim) == (2048, 128)
    bare = encoders.resnet50()
    assert isinstance(bare.fc, torch.nn.Linear) and [k for k in bare.state_dict() if k.startswith("fc.")] == \
        ["fc.weight", "fc.bias"]
    assert encoders.has_mlp_head(model.state_dict()) and not encoders.has_mlp_head(bare.state_dict())
    ref = encoders.to_reference_state_dict(model.state_dict())
    assert [k for k in ref if k.startswith("fc.")] == keys
    assert encoders.has_mlp_head({"module." + k: v for k, v in ref.items()})
    x = torch.randn(2, 3, 64, 64)
    model.eval()
    with torch.no_grad():
        feat = model(x, 6)
        want = model.fc[2](torch.relu(model.fc[0](feat)))
        assert torch.allclose(model(x), want / want.norm(dim=1, keepdim=True), atol=1e-6)
        model.l2norm = False
        assert torch.allclose(model(x), want, atol=1e-6)


def test_mlp_checkpoint_round_trips(tmp_path):
    from moco_b200.linear_eval import get_scheduler
    from moco_b200.NCE import MemoryMoCo
    model, ema = _mlp_state()
    contrast = MemoryMoCo(128, 64, 0.2)
    opt = torch.optim.SGD(model.parameters(), lr=0.03, momentum=0.9)
    sched = get_scheduler(opt, 2, 5, "cosine", 0, 100)
    args = _trainer("train_moco_v2_ckpt").parse_args(["--data-dir", "d", "--aug", "V2", "--mlp"])
    checkpoint.save(checkpoint.state(args, 1, model, ema, contrast, opt, sched), str(tmp_path), 1)
    ckpt = checkpoint.load(str(tmp_path / "current.pth"))
    assert ckpt["opt"]["mlp"] is True and ckpt["opt"]["aug"] == "V2"
    assert "module.fc.0.weight" in ckpt["model"] and "fc.2.bias" in ckpt["model_ema"]
    m2, e2 = encoders.resnet18(mlp=True), encoders.resnet18(mlp=True)
    opt2 = torch.optim.SGD(m2.parameters(), lr=0.03, momentum=0.9)
    assert checkpoint.restore(ckpt, m2, e2, MemoryMoCo(128, 64, 0.2), opt2) == 2
    for k, v in model.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k
    built = encoders.encoder_from_state_dict(ckpt["model"], "resnet18")     # the eval examples' builder
    assert isinstance(built.fc, torch.nn.Sequential)
    for k, v in model.state_dict().items():
        assert torch.equal(v, built.state_dict()[k]), k
    assert isinstance(encoders.encoder_from_state_dict(encoders.resnet18().state_dict(), "resnet18").fc,
                      torch.nn.Linear)
    with pytest.raises(RuntimeError):
        encoders.resnet18().load_state_dict(encoders.from_reference_state_dict(ckpt["model"]))


def test_reference_resnet50_refuses_an_mlp_checkpoint():
    """The documented deviation: the reference's eval.py strict-loads a bare-fc ResNet."""
    if not os.path.isfile(os.path.join(REF, "moco", "models", "resnet.py")):
        pytest.skip("oracle/_ref is not staged")
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import moco.models.resnet as ref_resnet
    sd = encoders.to_reference_state_dict(encoders.resnet50(mlp=True).state_dict())
    with pytest.raises(RuntimeError, match="fc"):
        ref_resnet.resnet50().load_state_dict(sd)
    ref_resnet.resnet50().load_state_dict(encoders.to_reference_state_dict(encoders.resnet50().state_dict()))
