"""MMGCF's late-fusion entry points refuse bad arguments before any CUDA call, in the C ABI and in `ops.late_fuse`, so
this runs without a GPU."""
import ctypes

import pytest
import torch


def test_c_entry_points_refuse_bad_arguments():
    from mmrec_b200 import _lib
    lib = _lib.load()
    P = 0x1000                                                           # a fake device address: nothing is dereferenced
    fwd = lib.mmrec_late_fuse_f32
    assert fwd(-1, 64, 0, 0, None, P, 10, P, None, None, P, None) == -1                  # negative n
    assert b"late_fuse" in lib.mmrec_last_error()
    assert fwd(8, 64, 2, 0, None, P, 10, P, None, None, P, None) == -1                   # fusion 2 (concat has no kernel)
    assert fwd(8, 64, 0, 3, None, P, 10, P, None, None, P, None) == -1                   # weighting 3
    assert fwd(8, 48, 0, 0, None, P, 10, P, None, None, P, None) == -4                   # d = 48: no kernel
    assert fwd(8, 64, 0, 0, None, P, 4, P, None, None, P, None) == -1                    # 8 rows without idx, E has 4
    assert fwd(8, 64, 0, 0, None, P, 10, None, None, None, P, None) == -1                # neither modality
    assert fwd(8, 64, 0, 1, None, P, 10, P, P, None, P, None) == -1                      # alpha weighting without alpha
    assert fwd(8, 64, 0, 0, None, P, 10, P, P, None, None, None) == -1                   # null out
    assert fwd(0, 64, 0, 0, None, None, 0, None, None, None, None, None) == 0            # nothing to do
    bwd = lib.mmrec_late_fuse_bwd_f32
    ws = lib.mmrec_late_fuse_workspace_bytes(8, 64)
    assert ws >= 8 and lib.mmrec_late_fuse_workspace_bytes(8, 48) == 0
    assert bwd(8, 64, 0, 0, None, P, 10, P, P, None, None, P, P, P, None, None, 0, None) == -1   # null g
    assert bwd(8, 64, 0, 0, None, P, 10, P, P, None, P, P, P, None, None, None, 0, None) == -1   # T given, dT null
    assert bwd(8, 64, 0, 1, None, P, 10, P, P, P, P, P, P, P, None, P, ws, None) == -1          # alpha without dalpha
    assert bwd(8, 64, 0, 1, None, P, 10, P, P, P, P, P, P, P, P, P, ws - 1, None) == -2         # workspace too small
    assert b"workspace" in lib.mmrec_last_error()


def test_ops_late_fuse_refuses_bad_arguments():
    from mmrec_b200 import ops
    from mmrec_b200._lib import MMRecError
    E, v = torch.zeros(10, 64), torch.zeros(10, 64)
    for kw in (dict(fusion="concat", weighting="equal"), dict(fusion="mean", weighting="gated"),
               dict(fusion="mean", weighting="alpha"),                                   # alpha weighting without alpha
               dict(fusion="mean", weighting="equal", alpha=torch.zeros(1))):             # alpha without alpha weighting
        with pytest.raises(MMRecError):
            ops.late_fuse(E, v, None, **kw)
    with pytest.raises(MMRecError):
        ops.late_fuse(E, None, None, "sum", "equal")                                      # neither modality
    with pytest.raises(MMRecError):
        ops.late_fuse(torch.zeros(10, 48), torch.zeros(10, 48), None, "sum", "equal")      # d = 48
    with pytest.raises(MMRecError):
        ops.late_fuse(E, torch.zeros(9, 64), None, "sum", "equal")                        # modality rows != item rows
    with pytest.raises(MMRecError):
        ops.late_fuse(E, torch.zeros(3, 64), None, "sum", "equal", idx=torch.arange(4))   # modality rows != len(idx)
    with pytest.raises(MMRecError):
        ops.late_fuse(E, v, None, "sum", "alpha", alpha=torch.zeros(2))                   # alpha of two elements
    if not torch.cuda.is_available():
        with pytest.raises(MMRecError):
            ops.late_fuse(E, v, None, "sum", "equal")                                     # CPU tensors: no CPU path
