"""CPU: the C-ABI library loads, exports exactly what include/lpb200.h declares, validates its
arguments, and the product path refuses to run without CUDA (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "lpb200.h")


def header_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lpb_[a-z0-9_]+)\s*\(", src)))


def test_header_is_plain_c():
    import subprocess

    subprocess.run(["gcc", "-fsyntax-only", "-x", "c", HEADER], check=True)


def test_library_exports_every_declared_symbol():
    from lightning_pose_b200 import _lib

    syms = header_symbols()
    assert len(syms) >= 19
    for s in syms:
        assert hasattr(_lib.lib, s), f"{s} declared in lpb200.h but not exported by liblpb200.so"
    assert sorted(_lib.SIGNATURES) == syms, "ctypes signature table out of sync with the header"
    assert _lib.lib.lpb_version() >= 200
    assert _lib.lib.lpb_build_arch() == b"sm_90a"


def test_decode_and_target_entries_validate_arguments_without_gpu():
    from lightning_pose_b200 import _lib

    rc = _lib.lib.lpb_decode_fwd(None, 1, 8, 8, 2, 1000.0, None, None, None, None, None)
    assert rc == -1 and b"null pointer" in _lib.lib.lpb_last_error()
    rc = _lib.lib.lpb_decode_prepare(8, 8, 7)
    assert rc == -1 and b"bad shape" in _lib.lib.lpb_last_error()
    with pytest.raises(_lib.LpbError):
        _lib.check(_lib.lib.lpb_generate_heatmaps(None, None, 1, 1.0, 1.0, 4, 4, 1.25, None, None))


def test_no_cpu_fallback():
    from lightning_pose_b200 import ops
    from lightning_pose_b200.losses.losses import HeatmapMSELoss, TemporalLoss
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead, run_subpixelmaxima

    x = torch.rand(1, 2, 8, 8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.decode_softargmax(x, 2, 1000.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        run_subpixelmaxima(x, 2, torch.tensor(1000.0))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        HeatmapHead("resnet50", 64, 5)(torch.rand(1, 64, 2, 2))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        HeatmapMSELoss()(heatmaps_targ=x, heatmaps_pred=x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        TemporalLoss()(torch.rand(4, 6))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "lightning_pose_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("# oracle", ""), f"{f} references the oracle"


def header_prototypes():
    """name -> number of parameters, parsed from the (comment-stripped) header."""
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(lpb_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S):
        args = m.group(2).strip()
        out[m.group(1)] = 0 if args in ("", "void") else len([a for a in args.split(",") if a.strip()])
    return out


def test_ctypes_table_matches_header_arity():
    """Every ctypes signature has exactly as many arguments as the C prototype it binds."""
    from lightning_pose_b200 import _lib

    protos = header_prototypes()
    assert sorted(protos) == header_symbols()
    for name, (_, argtypes) in _lib.SIGNATURES.items():
        assert len(argtypes) == protos[name], f"{name}: ctypes has {len(argtypes)} arguments, header has {protos[name]}"


def test_head_training_entry_points_validate_without_gpu():
    """The backward-side ABI (sizes, null checks) is callable without a GPU; nothing computes."""
    from lightning_pose_b200 import _lib

    n = ctypes.c_size_t(0)
    # saved shuffled features: B x (C/32) K-chunks x padded rows x 16 bytes (row layout: (2H)(2W+1) + 2(2W+2) rows, /8 up)
    assert _lib.lib.lpb_head_bf16_saved_bytes(3, 2048, 12, 12, ctypes.byref(n)) == 0
    rows = (24 * 25 + 2 * 26 + 7) // 8 * 8
    assert n.value == 3 * 64 * rows * 16
    assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes(3, 2048, 12, 12, 17, 17, ctypes.byref(n)) == 0
    rows2 = (48 * 49 + 2 * 50 + 7) // 8 * 8
    assert n.value >= 3 * 10 * (rows + rows2) * 16
    rc = _lib.lib.lpb_head_bwd_bf16(None, None, None, None, None, None, None, 1, 2048, 12, 12, None, 17, None, 17,
                                    None, None, None, None, None, None, None)
    assert rc == -1 and b"null pointer" in _lib.lib.lpb_last_error()
    rc = _lib.lib.lpb_decode_bwd_windows(None, None, None, 1, 8, 8, 2, 1000.0, None, None, None, None, None)
    assert rc == -1 and b"null pointer" in _lib.lib.lpb_last_error()


def test_decode_fwd_workspace_without_gpu():
    """The forward decode's scratch is the caller's: (2n + 1) ints of queue and arrival counters, then n x 16 x 4 floats of
    partial softmax states.  The size query needs no GPU, and lpb_decode_fwd refuses a missing or misaligned workspace
    before it queues anything (the other pointers are fake)."""
    from lightning_pose_b200 import _lib

    L = _lib.lib
    n = ctypes.c_size_t(0)
    for planes in (0, 1, 17, 768 * 17):
        assert L.lpb_decode_fwd_workspace_bytes(planes, ctypes.byref(n)) == 0
        assert n.value == 4 * (2 * planes + 1) + 4 * planes * 16 * 4
    assert L.lpb_decode_fwd_workspace_bytes(-1, ctypes.byref(n)) == -1
    assert L.lpb_decode_fwd_workspace_bytes(1, None) == -1
    fake = ctypes.c_void_p(0x1000)
    rc = L.lpb_decode_fwd(fake, 17, 96, 96, 2, 1000.0, fake, fake, fake, None, None)
    assert rc == -1 and L.lpb_last_error() == b"decode_fwd: null workspace"
    rc = L.lpb_decode_fwd(fake, 17, 96, 96, 2, 1000.0, fake, fake, fake, ctypes.c_void_p(0x1002), None)
    assert rc == -1 and L.lpb_last_error() == b"decode_fwd: workspace must be 4-byte aligned"


_BWD_VECTOR_BUFFERS = ["dfeat", "g_out", "probs", "win_meta", "g_overflow", "saved_xs", "fwd_workspace", "workspace"]


@pytest.mark.parametrize("misaligned", _BWD_VECTOR_BUFFERS)
def test_head_bwd_refuses_misaligned_buffers_without_gpu(misaligned):
    """lpb_head_bwd_bf16 moves these buffers with 16-byte vectors, bulk copies or TMA.  A pointer that is 2-byte but not
    16-byte aligned (0x1002) is refused with LPB_ERR_INVALID while the arguments are checked: the other pointers are fake,
    so a queued kernel or a CUDA call (LPB_ERR_CUDA without a GPU) would show here."""
    from lightning_pose_b200 import _lib

    p = {name: 0x1000 for name in _BWD_VECTOR_BUFFERS + ["win", "w1", "w2", "dw1", "db1", "dw2", "db2"]}
    p[misaligned] = 0x1002
    rc = _lib.lib.lpb_head_bwd_bf16(p["g_out"], p["probs"], p["win"], p["win_meta"], p["g_overflow"], p["saved_xs"], p["fwd_workspace"],
                                    3, 512, 8, 8, p["w1"], 9, p["w2"], 9, p["dfeat"], p["dw1"], p["db1"], p["dw2"], p["db2"], p["workspace"], None)
    assert rc == -1, (rc, _lib.lib.lpb_last_error())
    assert _lib.lib.lpb_last_error() == f"head_bwd_bf16: {misaligned} must be 16-byte aligned".encode()


@pytest.mark.parametrize("misaligned,addr,need", [("features", 0x1002, 16), ("saved_xs", 0x1008, 16), ("workspace", 0x1004, 16),
                                                   ("out", 0x1004, 8)])
@pytest.mark.parametrize("c,h,w,c2", [(2048, 12, 12, 17), (384, 16, 16, 0)])  # fast path, banded path
def test_head_fwd_refuses_misaligned_buffers_without_gpu(misaligned, addr, need, c, h, w, c2):
    """lpb_head_fwd_bf16 reads the features with TMA or 16-byte loads, moves saved_xs / workspace with bulk copies and
    writes out with 8-byte stores: a pointer short of that alignment is refused before anything is queued, on either
    kernel family."""
    from lightning_pose_b200 import _lib

    p = {name: 0x1000 for name in ("features", "w1", "b1", "w2", "b2", "out", "saved_xs", "workspace")}
    p[misaligned] = addr
    rc = _lib.lib.lpb_head_fwd_bf16(p["features"], 2, c, h, w, p["w1"], p["b1"], 17, p["w2"] if c2 else None, p["b2"] if c2 else None, c2, 1,
                                    p["out"], p["saved_xs"], p["workspace"], None)
    assert rc == -1, (rc, _lib.lib.lpb_last_error())
    assert _lib.lib.lpb_last_error() == f"head_fwd_bf16: {misaligned} must be {need}-byte aligned".encode()


def test_fused_head_node_refuses_cpu_tensors():
    from lightning_pose_b200.models.heads.heatmap import HeatmapHead

    head = HeatmapHead("resnet50", 64, 5)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        head.forward_with_keypoints(torch.rand(1, 64, 2, 2))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        head.forward_with_keypoints(torch.rand(1, 64, 2, 2).bfloat16())


def test_reference_arm_does_not_import_the_product():
    """bench.py --impl reference / cpu_baseline run the reference's own files (oracle/ref_arm.py); the arm must not load
    lightning_pose_b200 (or its .so) at all."""
    import subprocess
    import sys

    code = (
        "import sys, torch; sys.path.insert(0, %r); import bench\n"
        "from oracle.ref_arm import ReferenceStep\n"
        "bench.FEAT_C, bench.FEAT_HW, bench.IMG, bench.HM = 64, 4, 128, 32\n"
        "prob = bench.make_problem(1, 5, 'cpu', 'fresh')\n"
        "step = ReferenceStep(prob, 128, 32, bench.B_LABELED, bench.T_UNLABELED)\n"
        "v = step(True)\n"
        "assert torch.isfinite(v), v\n"
        "bad = [m for m in sys.modules if m.startswith('lightning_pose_b200')]\n"
        "assert not bad, bad\n"
        "print(step.kind)\n" % ROOT
    )
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    assert res.stdout.strip().splitlines()[-1] in ("reference", "port")
    # the staged copy (what the GPU box executes: it has no /root/reference) must be self-sufficient
    staged = os.path.join(ROOT, "oracle", "_ref")
    if os.path.isdir(os.path.join(staged, "lightning_pose")):
        res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env={**os.environ, "LP_REFERENCE_ROOT": staged})
        assert res.returncode == 0, res.stderr[-2000:]
        assert res.stdout.strip().splitlines()[-1] == "reference"


def test_round2_and_ws_backward_entries_validate_arguments_without_gpu():
    """Every entry added in round 2 rejects null / malformed arguments with an error code (never a crash), and the
    shape planner works without a device (callers size buffers with it)."""
    import ctypes as C

    from lightning_pose_b200 import _lib

    L = _lib.lib
    plan = C.c_int(-1)
    assert L.lpb_head_bf16_plan(2048, 12, 12, 17, 17, C.byref(plan)) == 0 and plan.value == 1   # cfg 2: whole-frame kernels
    assert L.lpb_head_bf16_plan(2048, 16, 16, 17, 17, C.byref(plan)) == 0 and plan.value == 0   # cfg 5: banded
    assert L.lpb_head_bf16_plan(384, 16, 16, 17, 0, C.byref(plan)) == 0 and plan.value == 0     # cfg 3: one deconv
    assert L.lpb_head_bf16_plan(384, 24, 24, 17, 0, C.byref(plan)) == 0 and plan.value == 0     # cfg 4
    assert L.lpb_head_bf16_plan(100, 12, 12, 17, 17, C.byref(plan)) == -1                          # C % 128
    assert L.lpb_head_bf16_plan(2048, 12, 12, 20, 17, C.byref(plan)) == -1                         # c1 must leave the ones channel
    n = C.c_size_t(0)
    assert L.lpb_head_bf16_workspace_bytes(2, 384, 16, 16, 17, 0, C.byref(n)) == 0 and n.value == 3 * 20480 + 20480 + 1792  # no mid for one deconv; + split-softmax statistics (2 frames x 5 bands x 20 x 2 floats, 256-byte aligned)
    assert L.lpb_head_bwd_bf16_workspace_bytes(2, 384, 16, 16, 17, 0, C.byref(n)) == 0 and n.value > 0
    for rc in (
        L.lpb_convt_fwd_f32(None, 1, 4, 4, 4, 1, None, None, 2, None, None),
        L.lpb_convt_bwd_f32_ws(None, None, 1, 4, 4, 4, 1, None, 2, None, None, None, None, 0, None),
        L.lpb_plane_softmax_f32(None, 1, 16, None),
        L.lpb_temporal_heatmap_loss_bwd(None, None, None, 4, 2, 8, 8, 0, None, 0.1, None, None, None),
        L.lpb_keypoints_mask_oob(None, 4, 64.0, 64.0, None, None),
        L.lpb_crnn_prepare(None, None, None, None, 5, 16, None, None, None),
        L.lpb_crnn_combine_fwd(None, None, None, 1, 5, 5, 8, 8, None, None, None, None, None, None),
        L.lpb_crnn_combine_bwd_ws(None, None, None, None, 1, 5, 5, 8, 8, None, None, None, None, None, None, None, None, None, None, None, 0, None),
        L.lpb_context_gather(None, 4, 64, 5, None, None),
        L.lpb_frames_normalize(None, 1, 8, 8, 8, 8, None, None, 0, 0, None, None),
        L.lpb_pack_predictions(None, None, 1, 2, None, 4, None, 0, None),
        L.lpb_adam_step(1, None, None, None, None, None, None, None, 1e-3, None, 0.9, 0.999, 1e-8, 0.0, 0, None),
        L.lpb_adam_step(17, C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), C.c_void_p(16), 1e-3, None, 0.9, 0.999, 1e-8, 0.0, 0, None),
        L.lpb_head_fwd_bf16(None, 1, 384, 16, 16, None, None, 17, None, None, 0, 1, None, None, None, None),
        L.lpb_head_bwd_bf16(None, None, None, None, None, None, None, 1, 384, 16, 16, None, 17, None, 0, None, None, None, None, None, None, None),
    ):
        assert rc == -1, (rc, L.lpb_last_error())
    assert L.lpb_context_gather(C.c_void_p(16), 4, 24, 5, C.c_void_p(16), None) == -1  # items must be 16-byte multiples
    assert L.lpb_context_gather_bwd(None, 4, 64, 5, 0, None, None) == -1
    assert L.lpb_context_gather_bwd(C.c_void_p(16), 4, 64, 4, 0, C.c_void_p(16), None) == -1  # odd context length
    assert L.lpb_context_gather_bwd(C.c_void_p(16), 4, 64, 5, 3, C.c_void_p(16), None) == -1  # no such element format


def test_tuning_switch_takes_only_softmax_split():
    """LPB_TUNE_SOFTMAX_SPLIT (key 7) is the one tuning switch: its default splits below one wave, and every other key
    is rejected by lpb_set_tuning and reads -1."""
    from lightning_pose_b200 import _lib

    L = _lib.lib
    assert L.lpb_set_tuning(99, 1) == -1 and L.lpb_get_tuning(99) == -1
    assert L.lpb_get_tuning(7) == 1
    for k in [*range(7), *range(8, 16)]:
        assert L.lpb_set_tuning(k, 1) == -1 and L.lpb_get_tuning(k) == -1


def test_head_shape_planner_python_side():
    from lightning_pose_b200 import ops

    ok = ops.head_bf16_supported
    assert ok((8, 2048, 12, 12), [17, 17], train=True) and ok((8, 2048, 16, 16), [17, 17], train=True)   # cfg 2, cfg 5
    assert ok((8, 384, 16, 16), [17], train=True) and ok((8, 384, 24, 24), [17], train=True)              # cfg 3, cfg 4
    assert not ok((8, 2048, 13, 13), [17, 17], train=False)      # H*W % 8
    assert not ok((8, 2048, 12, 12), [17, 17, 17], train=False)  # three deconvs: fp32 kernels
    assert not ok((8, 2048, 12, 12), [20, 17], train=False)      # no room for the ones channel
    assert ok((8, 512, 6, 4), [17, 17], train=False) and not ok((8, 512, 6, 20), [17, 17], train=True)  # width outside the dgrad epilogue set
    assert not ok((8, 384, 15, 16), [17], train=True) and ok((8, 384, 15, 16), [17], train=False)      # odd height: forward only

    # the backward's shape rule lives in the library: its workspace query refuses what lpb_head_bwd_bf16 would refuse
    from lightning_pose_b200 import _lib

    n = ctypes.c_size_t(0)
    unsupported = -3  # LPB_ERR_UNSUPPORTED
    assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes(8, 384, 15, 16, 17, 0, ctypes.byref(n)) == unsupported
    assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes(8, 512, 6, 20, 17, 17, ctypes.byref(n)) == unsupported
    for c, h, w, c2 in ((2048, 12, 12, 17), (2048, 16, 16, 17), (384, 16, 16, 0), (384, 24, 24, 0)):  # cfg 2, 5, 3, 4
        assert _lib.lib.lpb_head_bwd_bf16_workspace_bytes(8, c, h, w, 17, c2, ctypes.byref(n)) == 0 and n.value > 0
