"""noisynet_b200 -- H100 (sm_90a) implementation of NoisyNet's quantized-conv + analog-noise hot path.

Public surface (mirrors the reference's operator API, SURVEY.md section 8b):
    noisynet_b200.hardware_model : NoisyConv2d, NoisyLinear, QuantMeasure, UniformQuantize, AddNoise,
                                   add_noise_calculate_power, distort_tensor
    noisynet_b200.quant          : QuantMeasure, UniformQuantize
    noisynet_b200.ops            : raw C-ABI ops on CUDA tensors
    noisynet_b200.net            : NoisyNet (the CIFAR net of noisynet.py:326-695 on the boundary modules)
    noisynet_b200.dp             : one-process-per-GPU gradient all-reduce
The CUDA extension is mandatory; importing the ops without it raises (no CPU fallback).
"""
__version__ = "0.1.0"
