"""photon_b200 — a GPU-native federated LLM pre-training engine for the NVIDIA H100.

Capabilities follow relogu/photon (federated LocalSGD/FedOpt pre-training of
MPT decoder-only LLMs, centralised DDP training, Hydra-style config surface,
shm hand-off, server/client checkpoints) with the hot paths re-designed for
Hopper: hand-written sm_90a kernels (wgmma/TMA GEMMs and attention, fused
norm/loss/optimizer kernels) and in-kernel NVLink collectives for the round
reduce/broadcast and the DDP gradient all-reduce.
"""
__version__ = "0.1.0"
