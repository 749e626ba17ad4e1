"""H100-native (sm_90a) hot path of Instant-NGP behind the operator surface of kwea123/ngp_pl.

    ngp_pl_b200.vren               drop-in for the reference's pybind11 module `vren` (12 operators)
    ngp_pl_b200.tcnn               tinycudann-shaped modules (NetworkWithInputEncoding, Encoding, Network)
    ngp_pl_b200.models             NGP, render, the autograd Functions -- same names as the reference's `models`
    ngp_pl_b200.losses             NeRFLoss, DistortionLoss
    ngp_pl_b200.trainer.Trainer    the fused, CUDA-graph captured training step (+ NCCL / NVLink data parallelism)

Everything computes in ngp_pl_b200/libngp_b200.so (C ABI: include/ngp_b200.h; build: `python -m ngp_pl_b200.build`).
There is no CPU or PyTorch fallback.
"""
