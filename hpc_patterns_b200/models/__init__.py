"""The pattern programs of the suite (the "model families" a user of the reference looks for):
concurency (compute-while-copy overlap), peer2pear (P2P bandwidth + fused exchange), allreduce
miniapp (ring / collective), interop demos; tensor_parallel (beyond the reference: linear layers whose
collective is fused into the wgmma GEMM)."""
