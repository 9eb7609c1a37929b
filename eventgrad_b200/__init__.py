"""eventgrad_b200 — Hopper-native event-triggered decentralized SGD.

A from-scratch framework with the capabilities of soumyadipghosh/eventgrad
(centralized all-reduce SGD, ring D-PSGD gossip, EventGraD adaptive-threshold
event-triggered gossip and its top-k sparsified variant), designed for
8xH100 / NVLink 4: one process per GPU, parameters in a flat fp32 arena,
neighbour exchange + consensus average + SGD fused into hand-written sm_90a
kernels that store straight into peer memory.

Layout
------
models/    MLP, CNN-1/CNN-2, LeNet-CIFAR, ResNet family (reference + canonical)
data/      synthetic + real MNIST / CIFAR-10 sources, samplers, GPU augmentation
parallel/  ring topology, parameter arena, trigger FSM oracle, comm backends
ops/       Python front-ends of the CUDA extension (gossip, all-reduce, top-k, ...)
csrc/      CUDA / C++ sources (sm_90a)
engine/    trainer, evaluation, simulator
utils/     logging (reference-compatible files), timers, checkpoints, clocks
cli/       cent / decent / event / spevent entrypoints
"""
__version__ = "0.1.0"

from .config import TrainConfig  # noqa: F401
