"""Kernel-level timing of the forward phases on one GPU (CUDA events, warm, per-launch).
usage: python tools/kbench.py [N ...]"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import Weights, make_net, algorithmic_bytes_fwd
from dsmil_wsi_b200 import _lib
from dsmil_wsi_b200.sharded import CudaShardOps, milnet_params


def main():
    Ns = [int(a) for a in sys.argv[1:]] or [10000, 100000]
    dev = torch.device("cuda", 0)
    net = make_net(Weights(0), dev)
    lib = _lib.load()
    ops = CudaShardOps(milnet_params(net))
    tags = ["scores", "q_mlp", "attend", "finalize", "fused_sm90"]
    for N in Ns:
        x = torch.rand(N, 512, device=dev)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        for mode in ("forward", "phase1"):
            fn = (lambda: net(x)) if mode == "forward" else (lambda: ops.phase1(x, 0))
            with torch.no_grad():
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
                lib.dsmil_profile_enable(1)
                reps = 10
                for _ in range(reps):
                    flush.zero_()            # evict the bag from L2 between repetitions
                    fn()
                torch.cuda.synchronize()
                ms = (ctypes.c_double * 8)(); n = (ctypes.c_uint64 * 8)()
                lib.dsmil_profile_read(ms, n)
                lib.dsmil_profile_enable(0)
            per = {t: round(ms[i] / n[i] * 1e3, 2) for i, t in enumerate(tags) if n[i]}
            alg = algorithmic_bytes_fwd(N, 512, 2)
            print(f"N={N} {mode}: per-launch us {per}; HBM-roofline time for this bag {alg / 6575.1e9 * 1e6:.2f} us, "
                  f"tiles={-(-N // 128)}", flush=True)


if __name__ == "__main__":
    main()
