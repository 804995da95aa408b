"""CPU-side tests (no GPU): the C-ABI library loads and exports every symbol the header declares,
host logic of the Python mirror (permutation ids, pull plans, module state), and the
world_size-2 ShuffleBN plan over gloo.  No compute entry point is called here."""
import ctypes
import os
import re
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import moco_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "moco_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(moco_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from moco_b200 import _lib
    lib = _lib.load()
    names = _header_symbols()
    assert len(names) >= 15
    assert sorted(_lib.SIGNATURES) == names, "moco_b200/_lib.py and include/moco_b200.h disagree"
    raw = ctypes.CDLL(_lib.lib_path())                       # a second dlopen, independent of _lib's handle
    for n in names:
        assert ctypes.cast(getattr(raw, n), ctypes.c_void_p).value
        assert callable(getattr(lib, n))
    assert lib.moco_abi_version() == _lib.ABI_VERSION == 3
    assert lib.moco_nce_workspace_bytes(256, 128, 16384) > 0


def test_library_is_sm90a_native():
    """The shipped .so carries sm_90a SASS with wgmma / TMA / mbarrier instructions (no PTX JIT, no fallback arch)."""
    import shutil
    import subprocess
    from moco_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in sass and "sm_100" not in sass
    for mnemonic in ("HGMMA", "UTMALDG", "SYNCS", "UBLKCP"):
        assert mnemonic in sass, mnemonic


def test_error_reporting_without_gpu_is_loud():
    from moco_b200 import _lib
    lib = _lib.load()
    rc = lib.moco_nce_fwd(None, None, 0, None, 1, 64, 1, 1.0, None, None, None, None, None, None, None, 0, 0, None)
    assert rc == -1 and b"null pointer" in lib.moco_last_error()
    with pytest.raises(RuntimeError, match="moco_nce_fwd"):
        _lib.check(rc, "moco_nce_fwd")


def test_shuffle_ids_match_reference_and_do_not_touch_global_rng(golden_dir):
    from moco_b200.util import plan_forward, shuffle_ids_cpu
    ids = np.load(os.path.join(golden_dir, "shuffle_ids.npz"))
    torch.manual_seed(123)
    expect_next = torch.rand(3)
    torch.manual_seed(123)
    for key in [k for k in ids.files if k.startswith("fwd_")]:
        _, bsz, epoch = key.split("_")
        f, b = shuffle_ids_cpu(int(bsz), int(epoch))
        assert f.dtype == torch.int64 and b.dtype == torch.int64
        np.testing.assert_array_equal(f.numpy(), ids[key])
        np.testing.assert_array_equal(b.numpy(), ids["bwd_" + key[4:]])
    assert torch.equal(torch.rand(3), expect_next), "global RNG was clobbered"
    f, _ = shuffle_ids_cpu(8, 7)
    np.testing.assert_array_equal(plan_forward(f, 1, 2).numpy(), ids["fwd_8_7"][4:])


def test_memory_moco_constructor_matches_reference_contract():
    from moco_b200.NCE import MemoryMoCo
    torch.manual_seed(0)
    m = MemoryMoCo(128, 64, 0.07)
    torch.manual_seed(0)
    stdv = 1.0 / np.sqrt(128 / 3)
    expect = torch.rand(64, 128).mul_(2 * stdv).add_(-stdv)          # Contrast.py:16-17 under the same seed
    assert torch.equal(m.memory, expect)
    assert m.queue_size == 64 and m.temperature == 0.07 and m.index == 0
    assert sorted(m.state_dict().keys()) == ["memory", "params"]
    assert m.params.tolist() == [-1] and m.params.dtype == torch.int64
    assert abs(float(m.memory.abs().max()) - O.queue_init_bound(128)) < 1e-2


def test_cpu_tensors_fail_loudly_without_gpu():
    from moco_b200.NCE import MemoryMoCo
    m = MemoryMoCo(64, 32, 0.07)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.randn(4, 64), torch.randn(4, 64), torch.randn(4, 64))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.enqueue(torch.randn(4, 64))


def test_generic_criterion_definition_matches_oracle():
    from moco_b200.NCE import NCESoftmaxLoss, fused_prob
    x = torch.randn(16, 101) * 5
    assert abs(float(NCESoftmaxLoss()(x)) - O.nce_softmax_loss(x.numpy())) < 1e-5
    assert abs(float(fused_prob(x)) - O.prob_metric(x.numpy())) < 1e-6


def test_encoder_shapes_and_unit_norm():
    from moco_b200.encoders import resnet18
    net = resnet18(low_dim=128).eval()
    with torch.no_grad():
        y = net(torch.randn(2, 3, 224, 224))
    assert y.shape == (2, 128)
    assert torch.allclose(y.norm(dim=1), torch.ones(2), atol=1e-5)


# ------------------------------------------------------------------ world_size 2 over gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, n, epoch, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from moco_b200.util import DistributedShufle, plan_forward, shuffle_ids_cpu
    g = torch.Generator().manual_seed(100 + rank)
    x = torch.randn(n, 3, 4, 4, generator=g)
    fwd, bwd = shuffle_ids_cpu(n * world, epoch)
    # the rows this rank would PULL over NVLink: emulate peer memory with a gloo all_gather
    peers = [torch.zeros_like(x) for _ in range(world)]
    dist.all_gather(peers, x)
    src = plan_forward(fwd, rank, world)
    x_shuf = torch.stack([peers[int(gr) // n][int(gr) % n] for gr in src])
    feat = x_shuf.reshape(n, -1)[:, :16].contiguous()
    fpeers = [torch.zeros_like(feat) for _ in range(world)]
    dist.all_gather(fpeers, feat)
    feat_all = torch.stack([fpeers[int(gr) // n][int(gr) % n] for gr in bwd])
    assert torch.equal(DistributedShufle.get_local_id(fwd), src)
    ret[rank] = dict(x=x.numpy(), x_shuf=x_shuf.numpy(), binds=bwd.numpy(), feat=feat.numpy(),
                     feat_all=feat_all.numpy(), feat_local=feat_all[rank * n:(rank + 1) * n].numpy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,n,epoch,tag", [(2, 4, 7, "w2_n4_e7"), (4, 6, 2, "w4_n6_e2")])
def test_shuffle_pull_plan_world_gt1_gloo(golden_dir, world, n, epoch, tag):
    """The per-rank pull plan (which global rows each rank reads from which peer) reproduces the
    reference's all_gather+index ShuffleBN at world_size 2 and 4."""
    g = np.load(os.path.join(golden_dir, "shuffle.npz"))
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_gloo_worker, args=(world, n, epoch, _free_port(), ret), nprocs=world, join=True)
    for r in range(world):
        for key in ("x", "x_shuf", "binds", "feat", "feat_all", "feat_local"):
            np.testing.assert_array_equal(ret[r][key], g[f"{tag}_r{r}_{key}"], err_msg=f"rank {r} {key}")


def _shard_worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from moco_b200.NCE import ShardedMemoryMoCo
    torch.manual_seed(3)
    m = ShardedMemoryMoCo(128, 64, 0.07)
    mem0 = m.memory.numpy().copy()
    # checkpoint contract: state_dict() returns the FULL [K, C] queue by pulling the peers' shards, which needs the
    # shards peer-mapped (first step / share_memory_across_ranks, CUDA only) -- before that it must refuse loudly
    # rather than silently save 1/W of the queue
    try:
        m.state_dict()
        refused = False
    except RuntimeError as exc:
        refused = "peer-mapped" in str(exc)
    # load: a full [K, C] queue (reference / MemoryMoCo checkpoint) keeps this rank's block; a bare shard loads as is
    full = torch.arange(64 * 128, dtype=torch.float32).view(64, 128)
    m.load_state_dict({"params": torch.tensor([-1]), "memory": full})
    took_block = bool(torch.equal(m.memory, full[m.shard_row0:m.shard_row0 + m.shard_rows]))
    m.load_state_dict({"params": torch.tensor([-1]), "memory": full[:32] + 1})
    took_shard = bool(torch.equal(m.memory, full[:32] + 1))
    p = ShardedMemoryMoCo(128, 64, 0.07, persist_index=True)
    p.load_state_dict({"params": torch.tensor([40]), "memory": full})
    ret[rank] = dict(row0=m.shard_row0, rows=m.shard_rows, memory=mem0, refused=refused, took_block=took_block,
                     took_shard=took_shard, index=p.index, keys=sorted(k for k, _ in m.named_buffers()))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_queue_block_layout_world2_gloo():
    """ShardedMemoryMoCo host logic at world_size 2: rank r owns ring slots [r*K/W, (r+1)*K/W) and the shards
    concatenate to exactly the queue the reference's MemoryMoCo would have initialised under the same seed."""
    from moco_b200.NCE import MemoryMoCo
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_shard_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    torch.manual_seed(3)
    full = MemoryMoCo(128, 64, 0.07).memory.numpy()
    assert [ret[r]["row0"] for r in range(2)] == [0, 32] and all(ret[r]["rows"] == 32 for r in range(2))
    np.testing.assert_array_equal(np.concatenate([ret[0]["memory"], ret[1]["memory"]]), full)
    assert ret[0]["keys"] == ["memory", "memory_bf16", "params"]
    for r in range(2):
        assert ret[r]["refused"] and ret[r]["took_block"] and ret[r]["took_shard"] and ret[r]["index"] == 40
    with pytest.raises(ValueError, match="divisible"):
        # world size 1 here: any K is divisible, so emulate the check directly
        from moco_b200.NCE import ShardedContrast
        orig = ShardedContrast._world
        ShardedContrast._world = lambda: (0, 3)
        try:
            ShardedContrast.ShardedMemoryMoCo(128, 64, 0.07)
        finally:
            ShardedContrast._world = orig


def test_moment_update_has_no_cpu_fallback():
    """The EMA update is a CUDA kernel behind the C ABI; CPU parameters must raise, not silently run in torch."""
    import torch
    from moco_b200.util import moment_update
    a, b = torch.nn.Linear(4, 3), torch.nn.Linear(4, 3)
    before = b.weight.detach().clone()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        moment_update(a, b, 0.999)
    assert torch.equal(b.weight.detach(), before)
    moment_update(torch.nn.Identity(), torch.nn.Identity(), 0.5)      # no parameters: nothing to do


def test_persist_index_roundtrip_is_reference_compatible():
    """§8 f4: optional `index` persistence rides in the vestigial `params` buffer; keys/shapes unchanged."""
    import torch
    from moco_b200.NCE import MemoryMoCo
    ref_like = MemoryMoCo(8, 20, 0.07)                       # default: reference behaviour
    ref_like.index = 13
    sd = ref_like.state_dict()
    assert sorted(sd) == ["memory", "params"] and int(sd["params"]) == -1
    fresh = MemoryMoCo(8, 20, 0.07)
    fresh.load_state_dict(sd)
    assert fresh.index == 0                                  # the reference restarts the ring on resume

    a = MemoryMoCo(8, 20, 0.07, persist_index=True)
    a.index = 13
    sd = a.state_dict()
    assert sorted(sd) == ["memory", "params"] and sd["params"].shape == (1,) and int(sd["params"]) == 13
    b = MemoryMoCo(8, 20, 0.07, persist_index=True)
    b.load_state_dict(sd)
    assert b.index == 13 and torch.equal(b.memory, a.memory)
    b.load_state_dict(ref_like.state_dict())                 # a reference checkpoint: params == -1 -> index 0
    assert b.index == 0
    fresh.load_state_dict(sd)                                # reference-behaviour module ignores the value
    assert fresh.index == 0


def test_python_flag_constants_match_the_header():
    """moco_b200/_lib.py mirrors the MOCO_NCE_* / MOCO_GATHER_* enums and the one-pass temperature limit by hand."""
    import re
    from moco_b200 import _lib
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "moco_b200.h")).read()
    enum = {m.group(1): int(m.group(2)) for m in re.finditer(r"\b(MOCO_[A-Z0-9_]+)\s*=\s*(-?\d+)", text)}
    for name in ("AUTO", "FORCE_SIMT", "CTA_PAIR", "SINGLE_CTA", "TWO_PASS", "ONE_PASS"):
        assert getattr(_lib, "NCE_" + name) == enum["MOCO_NCE_" + name], name
    assert _lib.MOCO_F32 == enum["MOCO_F32"] and _lib.MOCO_BF16 == enum["MOCO_BF16"]
    limit = float(re.search(r"#define\s+MOCO_ONE_PASS_MAX_INV_T\s+([0-9.]+)f", text).group(1))
    assert _lib.ONE_PASS_MAX_INV_T == limit
    # every flag is a distinct bit
    bits = [enum["MOCO_NCE_" + n] for n in ("FORCE_SIMT", "CTA_PAIR", "SINGLE_CTA", "TWO_PASS", "ONE_PASS")]
    assert all(b & (b - 1) == 0 for b in bits) and len(set(bits)) == len(bits)


def test_example_trainer_accepts_every_launcher_spelling(monkeypatch):
    """SURVEY.md 8b: the reference's --local_rank only parser breaks under torch >= 2.0 launchers; the example
    entry point takes --local_rank, --local-rank and $LOCAL_RANK."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("train_moco_example", os.path.join(root, "examples", "train_moco.py"))
    mod = importlib.util.module_from_spec(spec)
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    spec.loader.exec_module(mod)
    assert mod.parse_args([]).local_rank == 0
    assert mod.parse_args(["--local_rank", "3"]).local_rank == 3
    assert mod.parse_args(["--local-rank=5"]).local_rank == 5
    monkeypatch.setenv("LOCAL_RANK", "6")
    assert mod.parse_args([]).local_rank == 6
    assert mod.parse_args(["--local-rank", "2"]).local_rank == 2
    a = mod.parse_args(["--nce-k", "65536", "--nce-t", "0.2", "--persist-index", "--fuse-normalize", "--graph-tail"])
    assert (a.nce_k, a.nce_t, a.persist_index, a.fuse_normalize, a.graph_tail) == (65536, 0.2, True, True, True)


def test_batchnorm_act_module_is_a_batchnorm2d_off_the_gpu():
    """BatchNormAct2d away from its kernels (CPU tensors here) = the reference's BatchNorm2d -> += residual -> ReLU
    (moco/models/resnet.py:96-102), with nn.BatchNorm2d's parameters, buffers and state_dict keys."""
    import torch.nn.functional as F
    from moco_b200.bn import BatchNormAct2d
    torch.manual_seed(0)
    m, r = BatchNormAct2d(8, relu=True), torch.nn.BatchNorm2d(8)
    x, res = torch.randn(4, 8, 5, 5), torch.randn(4, 8, 5, 5)
    assert torch.equal(m(x, res), F.relu(r(x) + res))
    assert torch.equal(m.running_var, r.running_var) and int(m.num_batches_tracked) == 1
    assert list(m.state_dict()) == list(r.state_dict())
    assert isinstance(m, torch.nn.BatchNorm2d)
    plain = BatchNormAct2d(8)
    assert torch.equal(plain(x), torch.nn.BatchNorm2d(8)(x))


def test_encoder_layout_is_unchanged_by_the_fused_norm_modules():
    """The BatchNormAct2d / MaxPool3x3s2 swap keeps ResNet-50's 161 parameter tensors (the EMA pairs of
    moco/util.py:124-127), their order, and the checkpoint keys of a plain conv / BatchNorm2d network."""
    from moco_b200 import encoders
    m = encoders.resnet50(128)
    assert len(list(m.parameters())) == 161 and sum(p.numel() for p in m.parameters()) == 23770304
    keys = set(m.state_dict())
    for k in ("stem.0.weight", "stem.1.running_mean", "stem.1.num_batches_tracked", "layers.0.bn3.weight",
              "layers.0.short.1.running_var", "layers.15.conv3.weight", "fc.bias"):
        assert k in keys, k
    assert not any(k.startswith("stem.2") or k.startswith("stem.3") for k in keys)


def test_bn_and_pool_entries_validate_their_arguments_without_a_gpu():
    from moco_b200 import _lib
    lib = _lib.load()
    assert lib.moco_bn_workspace_bytes() >= 256 + 128 * 4
    rc = lib.moco_bn_fwd_train(None, None, None, 1024, 64, None, None, None, None, None, 0.1, 1e-5, 1, None, None, None, 0, None)
    assert rc == -1 and b"moco_bn_fwd_train" in lib.moco_last_error()
    rc = lib.moco_bn_bwd(None, None, None, 1024, 64, None, None, None, None, 1, 1, None, None, None, None, None, 0, None)
    assert rc == -1 and b"moco_bn_bwd" in lib.moco_last_error()
    assert lib.moco_maxpool3x3s2_fwd(None, None, None, 1, 8, 8, 64, None) == -1
    assert lib.moco_maxpool3x3s2_bwd(None, None, None, 1, 8, 8, 64, None) == -1


# Addresses that are never dereferenced: every call below must return before it touches the device.
_A, _WS = 0x7f0000001000, 0x7f0000100000          # 16-byte / 256-byte aligned


@pytest.mark.parametrize("bad", ["q", "queue"])
def test_nce_fwd_rejects_misaligned_operands_without_a_gpu(bad):
    """q and the queue are read with 16-byte vector loads (TMA / uint4 rows): a contiguous view at an odd storage
    offset must be refused before any device access, not handed to a kernel that would fault."""
    from moco_b200 import _lib
    lib = _lib.load()
    ptr = {"q": _A, "queue": _A + 0x10000}
    ptr[bad] += 8
    args = lambda ws_bytes: (ptr["q"], _A + 0x20000, _lib.MOCO_BF16, ptr["queue"], 4, 64, 16, 1 / 0.07, None,
                             _A + 0x30000, _A + 0x30100, _A + 0x30200, _A + 0x30300, _A + 0x40000, _WS, ws_bytes, 0, None)
    rc = lib.moco_nce_fwd(*args(1 << 30))
    assert rc == -1 and b"16-byte aligned" in lib.moco_last_error(), lib.moco_last_error()
    ptr[bad] -= 8                                 # control: aligned, the next check (workspace size) answers
    assert lib.moco_nce_fwd(*args(0)) == -3


@pytest.mark.parametrize("bad", ["q", "queue", "queue_f32", "k_all"])
def test_nce_step_rejects_misaligned_operands_without_a_gpu(bad):
    from moco_b200 import _lib
    lib = _lib.load()
    ptr = {"q": _A, "queue": _A + 0x10000, "queue_f32": _A + 0x20000, "k_all": _A + 0x50000}
    ptr[bad] += 4
    args = lambda ws_bytes: (ptr["q"], _A + 0x60000, _lib.MOCO_F32, 0, ptr["queue"], ptr["queue_f32"], 4, 64, 16,
                             1 / 0.07, ptr["k_all"], _lib.MOCO_F32, 4, 3, None, _A + 0x30000, _A + 0x30100,
                             _A + 0x30200, _A + 0x30300, _A + 0x40000, _WS, ws_bytes, 0, None)
    rc = lib.moco_nce_step(*args(1 << 30))
    assert rc == -1 and b"16-byte aligned" in lib.moco_last_error(), lib.moco_last_error()
    ptr[bad] -= 4
    assert lib.moco_nce_step(*args(0)) == -3


@pytest.mark.parametrize("bad", ["queue", "queue_f32", "k_all"])
def test_enqueue_entries_reject_misaligned_operands_without_a_gpu(bad):
    """enqueue_kernel reads k_all and writes both queue copies 16 bytes at a time."""
    from moco_b200 import _lib
    lib = _lib.load()
    ptr = {"queue": _A, "queue_f32": _A + 0x10000, "k_all": _A + 0x20000}
    ptr[bad] += 2
    rc = lib.moco_queue_enqueue(ptr["queue"], ptr["queue_f32"], ptr["k_all"], _lib.MOCO_BF16, 4, 64, 16, 3, None)
    assert rc == -1 and b"moco_queue_enqueue: the queue and k_all must be 16-byte aligned" in lib.moco_last_error()
    rc = lib.moco_queue_enqueue_shard(ptr["queue"], ptr["queue_f32"], ptr["k_all"], _lib.MOCO_BF16, 4, 64, 16, 3, 0, 8,
                                      None)
    assert rc == -1 and b"moco_queue_enqueue_shard: the shard and k_all must be 16-byte aligned" in lib.moco_last_error()


def test_memory_moco_copies_a_misaligned_view_before_the_kernels_see_it():
    """A contiguous view at an odd storage offset passes .contiguous() unchanged; MemoryMoCo copies it instead."""
    from moco_b200.NCE.Contrast import _aligned16
    base = torch.zeros(1 + 4 * 64)
    view = base[1:].view(4, 64)
    assert view.is_contiguous() and view.data_ptr() % 16 != 0
    fixed = _aligned16(view)
    assert fixed.data_ptr() % 16 == 0 and torch.equal(fixed, view)
    ok = torch.zeros(4, 64)
    assert _aligned16(ok) is ok


def _launch_statement_end(src, i):
    """Index just past the `;` of the `<<<...>>>(...);` statement whose `<<<` is at i."""
    i = src.index(">>>", i) + 3
    depth = 0
    while True:
        depth += {"(": 1, ")": -1}.get(src[i], 0)
        i += 1
        if depth == 0 and src[i - 1] == ")":
            return src.index(";", i) + 1


def test_every_kernel_launch_is_counted():
    """moco_launch_count() is right only if every kernel launch in csrc/ is counted where it happens: each
    `<<<...>>>(...);` is followed by launched() before the next launch or return (a launch in the if-branch of an
    if / else is covered by the check after the else-branch), and the only launch API called, cudaLaunchKernelEx,
    is called inside counted() (launch_pdl, launch_cluster)."""
    csrc = os.path.join(ROOT, "moco_b200", "csrc")
    chevrons = launch_api = 0
    for name in sorted(os.listdir(csrc)):
        if not name.endswith((".cu", ".cuh")):
            continue
        src = re.sub(r"//[^\n]*|/\*.*?\*/", lambda m: "\n" * m.group().count("\n"),
                     open(os.path.join(csrc, name)).read(), flags=re.S)
        for m in re.finditer(r"<<<", src):
            chevrons += 1
            rest = src[_launch_statement_end(src, m.start()):]
            if re.match(r"\s*}?\s*else\b", rest):
                continue
            after = re.search(r"launched\(\)|<<<|\breturn\b(?!\s+launched\(\))", rest)
            where = f"{name}:{src.count(chr(10), 0, m.start()) + 1}"
            assert after and after.group() == "launched()", f"{where}: launch not followed by launched()"
        for m in re.finditer(r"\bcu(?:da)?Launch\w*\s*\(", src):
            launch_api += 1
            assert m.group().startswith("cudaLaunchKernelEx") and re.search(r"counted\(\s*$", src[:m.start()]), \
                f"{name}:{src.count(chr(10), 0, m.start()) + 1}: {m.group()} outside counted()"
    assert chevrons >= 30 and launch_api >= 2
