"""The C-ABI shared library loads here (no GPU) and exports every symbol include/mmrec_b200.h declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "mmrec_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(mmrec_[a-z0-9_]+)\s*\(", src)))


def test_library_built_and_exports_every_header_symbol():
    from mmrec_b200 import _lib
    assert os.path.isfile(_lib.LIB_PATH), "run __graft_entry__.build() first"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = header_functions()
    assert len(names) >= 17
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    assert set(names) == set(_lib.PROTOTYPES), "python prototypes and header disagree"


def test_loader_binds_and_reports_abi_version():
    from mmrec_b200 import _lib
    lib = _lib.load()
    assert lib.mmrec_abi_version() == _lib.ABI_VERSION == 4
    assert lib.mmrec_last_error() is not None


def test_argument_errors_before_any_cuda_call():
    """Argument validation happens before any CUDA call, so it is testable on a CPU box."""
    from mmrec_b200 import _lib
    lib = _lib.load()
    op = _lib.SpmmOp(n_rows=-1, ldx=64, ldy=64, ldacc=64, acc_div=1.0)
    assert lib.mmrec_spmm_run_f32(64, 1, ctypes.byref(op), 0, None) == -1
    assert b"spmm" in lib.mmrec_last_error()
    assert lib.mmrec_spmm_run_f32(64, 0, ctypes.byref(op), 0, None) == -1                  # no ops
    assert lib.mmrec_spmm_run_f32(64, 1, None, 0, None) == -1
    # well-formed ops on fake, 16-byte aligned addresses with a work plan: rejected before any CUDA call
    fake = dict(n_rows=8, n_cols=8, rowptr=0x1000, colidx=0x2000, vals=0x3000, tasks=0x4000, n_tasks=8, n_cta_tasks=0,
                split_rows=0x5000, counters=0x6000, partial=0x7000, Y=0x8000, ldy=48, acc_div=1.0)
    op = _lib.SpmmOp(X=0x9000, ldx=48, keep_bits=0xa000, keep_scale=1.0, **fake)
    assert lib.mmrec_spmm_run_f32(48, 1, ctypes.byref(op), 0, None) == -4                 # edge-keep mask at d = 48
    ops = (_lib.SpmmOp * 2)(_lib.SpmmOp(X=0x9000, ldx=64, **dict(fake, ldy=64)),
                            _lib.SpmmOp(X=0x9000, ldx=64, gate_ref=0xa000, ldgate=64, **dict(fake, ldy=64)))
    assert lib.mmrec_spmm_run_f32(64, 2, ops, 0, None) == -4                               # the chained kernel has no gate
    assert lib.mmrec_topk_rows_f32(4, 10, None, 10, 11, 0, None, None, None) == -1     # k > n_items
    assert lib.mmrec_project_f32(-5, None, None, 0, 0, None, None, 0, 0, None, 0, None, 0, None) == -1
    assert lib.mmrec_topk_merge(100, 4, 50, None, None, None, None, None) == -1        # parts * k > 4096
    # K4, peer-memory exchange: world out of range, n not a multiple of 4 floats, null list pointers
    two = (ctypes.c_void_p * 2)(16, 32)
    assert lib.mmrec_peer_sum_f32(8, 0, ctypes.cast(two, ctypes.c_void_p), None, None, 1.0, None, None) == -1
    assert lib.mmrec_peer_sum_f32(6, 2, ctypes.cast(two, ctypes.c_void_p), None, None, 1.0, None, None) == -1
    assert b"peer_sum" in lib.mmrec_last_error()
    assert lib.mmrec_topk_merge_peers(17, 4, 10, ctypes.cast(two, ctypes.c_void_p), ctypes.cast(two, ctypes.c_void_p), 1, 0, 0, 4,
                                      None, None, None, None, 0, None) == -1           # more than 16 lists
    assert lib.mmrec_topk_merge_peers(2, 4, 10, ctypes.cast(two, ctypes.c_void_p), ctypes.cast(two, ctypes.c_void_p), 2, 1, 3, 2,
                                      None, None, None, None, 0, None) == -1           # row range outside the batch
    assert lib.mmrec_topk_merge_peers(2, 0, 10, ctypes.cast(two, ctypes.c_void_p), ctypes.cast(two, ctypes.c_void_p), 2, 1, 0, 0,
                                      None, None, None, None, 0, None) == 0            # B == 0: nothing to do
    assert lib.mmrec_peer_reduce_push_f32(8, 2, 2, ctypes.cast(two, ctypes.c_void_p), ctypes.cast(two, ctypes.c_void_p), None, None, 1.0, 0,
                                          None) == -1                                  # rank outside the world
    assert lib.mmrec_peer_gather_f32(6, 2, ctypes.cast(two, ctypes.c_void_p), None, None) == -1
    assert lib.mmrec_catalog_bytes(7000, 64) >= 7000 * 64 * 2 and lib.mmrec_catalog_bytes(7000, 300) == 0
    assert lib.mmrec_launch_count() >= 0
    # f1: projection backward / Adam
    assert lib.mmrec_index_sum_rows_f32(4, None, None, 64, 300, 10, None, 300, None) == -1          # null pointers
    assert lib.mmrec_linear_wgrad_f32(8, None, None, 64, 64, None, 8, 4098, None, None, None, 0, None) == -1   # null pointers
    assert b"linear_wgrad" in lib.mmrec_last_error()
    assert lib.mmrec_linear_dgrad_f32(8, None, 200, 200, None, 4096, None, None) == -1
    assert lib.mmrec_linear_dgrad_adam_f32(8, 16, 200, 200, 32, 4096, None, None, None, 0.9, 0.999, 1e-8, 0.0, -1e-3, 1.0, None) == -4   # d > 128: no fused kernel
    assert lib.mmrec_linear_dgrad_adam_f32(0, None, 64, 64, None, 4096, None, None, None, 0.9, 0.999, 1e-8, 0.0, -1e-3, 1.0, None) == 0
    assert lib.mmrec_adam_f32(0, None, 0.9, 0.999, 1e-8, 0.0, None) == 0
    bad = (_lib.AdamTensor * 1)()
    bad[0].n, bad[0].bc2_sqrt = 16, 1.0                                                             # null pointers
    assert lib.mmrec_adam_f32(1, ctypes.cast(bad, ctypes.c_void_p), 0.9, 0.999, 1e-8, 0.0, None) == -1
    assert lib.mmrec_linear_wgrad_workspace_bytes(7000, 4096, 64) >= 64 * 4096 * 4


def test_product_path_refuses_cpu_tensors():
    import torch
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    with pytest.raises(MMRecError):
        ops.score(torch.zeros(4, 64), torch.zeros(8, 64))
    with pytest.raises(MMRecError):
        ops.CSR.from_coo(torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.int64), None, 4, 4)


def test_fused_adam_refuses_cpu_parameters():
    import torch
    from mmrec_b200.optim import FusedAdam
    from mmrec_b200._lib import MMRecError
    p = torch.nn.Parameter(torch.zeros(4))
    opt = FusedAdam([p], lr=1e-3)
    p.grad = torch.ones(4)
    with pytest.raises(MMRecError):
        opt.step()
    assert opt.state_dict()["param_groups"][0]["betas"] == (0.9, 0.999)


def test_product_never_imports_the_oracle():
    import subprocess, sys
    out = subprocess.run([sys.executable, "-c",
                          "import sys; sys.path.insert(0, %r); import mmrec_b200.ops, mmrec_b200.graph, "
                          "mmrec_b200.models.freedom, mmrec_b200.models.bm3, mmrec_b200.models.mgcn, "
                          "mmrec_b200.models.lightgcn, mmrec_b200.models.layergcn, mmrec_b200.models.mmgcn, mmrec_b200.sharded, "
                          "mmrec_b200.common.trainer, mmrec_b200.utils.quick_start, mmrec_b200.optim; "
                          "print(any(m == 'oracle' or m.startswith('oracle.') for m in sys.modules))" % ROOT],
                         capture_output=True, text=True, check=True)
    assert out.stdout.strip() == "False"
    for dirpath, _, files in os.walk(os.path.join(ROOT, "mmrec_b200")):
        for f in files:
            if f.endswith(".py"):
                assert "import oracle" not in open(os.path.join(dirpath, f)).read().replace("mmrec_oracle", "")
                assert "from oracle" not in open(os.path.join(dirpath, f)).read()
