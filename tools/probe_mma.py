"""Issue rate of wgmma as this library issues it (one warpgroup, both operands in shared memory, K-major no swizzle, M = 64):
    python tools/probe_mma.py
cycles per instruction and MACs per cycle and SM for tf32 / bf16 at N = 64 / 128 / 256."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mmrec_b200 import _lib
lib = _lib.load(); dev = torch.device("cuda:0")
out = torch.zeros(256, dtype=torch.int64, device=dev)
st = torch.cuda.current_stream().cuda_stream
for kind, name, K in ((0, "tf32", 8), (1, "bf16", 16)):
    for N in (64, 128, 256):
        for distinct in (0, 4):
            for iters in (256, 2048):
                assert lib.mmrec_debug_mma_rate(kind, N, iters, distinct, out.data_ptr(), st) == 0
                torch.cuda.synchronize()
                c = out[:torch.cuda.get_device_properties(dev).multi_processor_count].double().median().item()
            cyc = (c - 0) / 2048
            print(f"{name} M64 N{N:3d} K{K:2d} ({'lean issue loop' if distinct == 0 else 'descriptors rebuilt per MMA'}): {cyc:7.1f} cycles/MMA  {64 * N * K / cyc:7.0f} MAC/cycle/SM")
