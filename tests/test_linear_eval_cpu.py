"""Linear evaluation against the reference's own models (staged unmodified in oracle/_ref), on the CPU in fp32: the
checkpoint key mapping in both directions, ``MoCoResNet.forward(x, layer)`` against ``ResNet.forward(x, layer)``, and
``LinearClassifierResNet`` against the reference's classifier."""
import os
import sys

import pytest
import torch

from moco_b200 import encoders
from moco_b200.linear_eval import LinearClassifierResNet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


@pytest.fixture(scope="module")
def ref():
    if not os.path.isfile(os.path.join(REF, "moco", "models", "resnet.py")):
        pytest.skip("oracle/_ref is not staged (run __graft_entry__.build() where the reference checkout exists)")
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import moco.models.resnet as resnet
    import moco.models.LinearModel as linear
    return resnet, linear


def _randomise(model, seed):
    """Non-trivial BatchNorm parameters and running statistics, so that eval mode is not the identity."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                C = m.num_features
                m.weight.copy_(torch.rand(C, generator=g) + 0.5)
                m.bias.copy_(torch.randn(C, generator=g) * 0.2)
                m.running_mean.copy_(torch.randn(C, generator=g) * 0.3)
                m.running_var.copy_(torch.rand(C, generator=g) + 0.5)
                m.num_batches_tracked.fill_(int(torch.randint(1, 1000, (1,), generator=g)))


@pytest.mark.parametrize("arch", ["resnet18", "resnet34", "resnet50"])
def test_state_dict_key_mapping_round_trips(ref, arch):
    resnet, _ = ref
    torch.manual_seed(0)
    theirs = getattr(resnet, arch)()
    ours = getattr(encoders, arch)()
    _randomise(theirs, 1)
    sd_ref = theirs.state_dict()
    # same entries in the same order, names aside
    mapped = encoders.from_reference_state_dict(sd_ref)
    assert list(mapped) == list(ours.state_dict())
    ours.load_state_dict(mapped, strict=True)
    back = encoders.to_reference_state_dict(ours.state_dict())
    assert list(back) == list(sd_ref)
    assert all(torch.equal(back[k], sd_ref[k]) for k in sd_ref)
    theirs2 = getattr(resnet, arch)()
    theirs2.load_state_dict(back, strict=True)
    # the module. prefix of a DistributedDataParallel checkpoint (train.py saves model.state_dict() of the DDP wrapper)
    ddp = {"module." + k: v for k, v in sd_ref.items()}
    assert list(encoders.from_reference_state_dict(ddp)) == list(mapped)
    assert list(encoders.to_reference_state_dict({"module." + k: v for k, v in ours.state_dict().items()})) == list(sd_ref)
    # a state_dict already in this package's naming passes through
    assert list(encoders.from_reference_state_dict(ours.state_dict())) == list(ours.state_dict())


def test_forward_layer_matches_the_reference_forward_layer(ref):
    resnet, _ = ref
    torch.manual_seed(0)
    theirs = resnet.resnet50().eval()
    _randomise(theirs, 2)
    ours = encoders.resnet50()
    ours.load_state_dict(encoders.from_reference_state_dict(theirs.state_dict()))
    ours.eval()
    x = torch.randn(2, 3, 224, 224)
    with torch.no_grad():
        for k in range(0, 8):
            a, b = ours(x, layer=k), theirs(x, layer=k)
            assert a.shape == b.shape, k
            err = float((a - b).abs().max())
            assert err <= 1e-4 * float(b.abs().max()) + 1e-6, (k, err)
        assert torch.equal(ours(x), ours(x, 7))


def test_frozen_model_on_the_cpu_is_the_eval_model():
    torch.manual_seed(0)
    a = encoders.resnet18()
    _randomise(a, 3)
    b = encoders.resnet18()
    b.load_state_dict(a.state_dict())
    assert b.freeze() is b
    a.eval()
    assert not any(p.requires_grad for p in b.parameters()) and not b.training
    assert all(m.frozen for m in b.modules() if isinstance(m, encoders.BatchNormAct2d))
    assert list(b.state_dict()) == list(a.state_dict())
    x = torch.randn(2, 3, 64, 64)
    with torch.no_grad():
        for k in (1, 3, 5, 6, 7):
            assert torch.equal(a(x, k), b(x, k)), k


@pytest.mark.parametrize("layer", [1, 2, 3, 4, 5, 6])
def test_linear_classifier_matches_the_reference(ref, layer):
    _, linear = ref
    torch.manual_seed(layer)
    theirs = linear.LinearClassifierResNet(layer, 10, "avg", 1)
    ours = LinearClassifierResNet(layer, 10, "avg", 1)
    sd = theirs.state_dict()
    assert [(k, v.shape) for k, v in ours.state_dict().items()] == [(k, v.shape) for k, v in sd.items()]
    assert [n for n, _ in ours.named_modules()] == [n for n, _ in theirs.named_modules()]
    w = ours.classifier.LiniearClassifier.weight
    assert abs(float(w.detach().std()) - 0.01) < 2e-3 and float(ours.classifier.LiniearClassifier.bias.abs().max()) == 0.0
    ours.load_state_dict(sd)
    side = {1: 56, 2: 56, 3: 28, 4: 14, 5: 7}
    C = {1: 64, 2: 256, 3: 512, 4: 1024, 5: 2048, 6: 2048}[layer]
    if layer == 1:
        C = 128        # LinearModel.py:18 sizes layer 1 for 128 channels
    shape = (3, C) if layer == 6 else (3, C, side[layer], side[layer])
    feat = torch.randn(shape)
    want = theirs(feat)
    assert torch.allclose(ours(feat), want, rtol=1e-5, atol=1e-6)
    if layer < 6:
        got = ours(feat.contiguous(memory_format=torch.channels_last))
        assert torch.allclose(got, want, rtol=1e-5, atol=1e-6)
    with pytest.raises(NotImplementedError):
        LinearClassifierResNet(7)


def test_default_forward_still_runs_the_trunk_as_one_sequential():
    """forward(x) / forward(x, 6) of a model that is not frozen call ``layers`` as before: hooks on it fire, and the
    last block returns its map."""
    torch.manual_seed(0)
    m = encoders.resnet18().eval()
    seen = []
    m.layers.register_forward_hook(lambda mod, inp, out: seen.append(("layers", out.dim())))
    m.layers[-1].register_forward_hook(lambda mod, inp, out: seen.append(("last", out.dim())))
    with torch.no_grad():
        m(torch.randn(1, 3, 64, 64))
        m(torch.randn(1, 3, 64, 64), 6)
    assert seen == [("last", 4), ("layers", 4)] * 2
