"""Bounds of tests/test_update_recompute_bench_size_gpu.py, in a module of their own so that the CPU check of the planted
defects (tests/test_update_fallback_reference_cpu.py) can use them without importing a GPU test file.

Each bound is about 3x the worst value seen on an H100 80GB HBM3 (400 W power limit); the observed values are given
beside it."""

# whole recompute update, G rel-L2 overall and worst named tensor.  Observed with TF32 allowed (the bench default):
# overall 3.7e-4 / 2.4e-4 / 3.0e-4 (grid / Monaco / IA2C), 3.6e-4 (grid R = 2500), worst tensor 4.7e-4 (wh); with fp32
# products: overall 7.6e-5 / 2.7e-5 / 7.2e-5, worst tensor 9.1e-5 (wx).  TF32 rounds the forward's X . Wx product too,
# which the float64 reference cannot restate: that is the gap between the two.
RECOMPUTE_G_REL_L2 = 1.2e-3
RECOMPUTE_TENSOR_REL_L2 = 1.5e-3
RECOMPUTE_G_REL_L2_FP32 = 2.5e-4
RECOMPUTE_TENSOR_REL_L2_FP32 = 3e-4
# whole FcACPolicy update, G rel-L2 overall; fp32 tensors (wx, bl, wo, bo) and fc front-end tensors, worst rel-L2.
# Observed: overall 3.9e-5, fp32 tensors 1.2e-5 (wx), fc front end 8.0e-5 (fct_w)
FC_G_REL_L2 = 1.2e-4
FC_FP32_TENSOR_REL_L2 = 4e-5
FC_FRONT_TENSOR_REL_L2 = 2.5e-4
# kernels, max |delta| / max |ref| of each output.  fp32 SIMT kernels (fc_embed, lstm_seq_fwd, fc_hidden_fwd / bwd):
# observed 9.4e-7 at most (lstm_seq_fwd gates); heads_loss with fp32 H: dH 5.3e-7, wo 9.9e-7, bo 3.2e-5 (the bias sums
# cancel), the bounds of the store-path test; FC forward: pi 2.0e-6, value 4.8e-7
FP32_KERNEL_MAX = 2.5e-6
HEADS_MAX = {"dH": 2e-6, "wo": 3e-6, "bo": 1e-4}
FC_FORWARD_MAX = 6e-6
# tensor-core kernels on fp32 operands converted to bf16: wgrad_tc_kernel 1.3e-4, fc_bwd_tc_kernel 6.8e-5
WGRAD_FP32_MAX = 4e-4
FC_BWD_FP32_MAX = 2e-4
# lstm_bwd_tc_kernel<512> on fp32 gates / c vs bptt_ref, dz_errors: rel-L2 6.9e-5, max 9.9e-4 (grid, Monaco, Rc = 1000).
# The six planted defects of bptt_mutations move it by 0.32 (c0 row) to 1.42 (dH shifted)
BPTT_FP32_REL_L2 = 2e-4
BPTT_FP32_MAX = 3e-3
