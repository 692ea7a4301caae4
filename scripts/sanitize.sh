#!/bin/bash
# Memory-checking tier (the reference has none, SURVEY.md §5): a subset of the GPU kernel tests
# under compute-sanitizer memcheck. The fused kernel runs with W virtual ranks on ONE GPU, so every
# global / "peer" access, the TMA bulk copies and the mbarrier of the item cache are covered.
# (racecheck only tracks shared memory; the kernels synchronise through global flags, and the one
# shared structure -- the item cache -- is written by TMA before a barrier and read-only afterwards.)
set -e
cd "$(dirname "$0")/.."
SUBSET='test_fused_sra_tiny_and_exact_constant or (test_fused_sra_matches_cpu_oracle and 4-dtype0) or test_fused_sra_mixed_layers_unaligned or (test_quantize_kernel_bytes_match_cpu and dtype0-4-512) or (test_oneshot_kernel_matches_cpu_oracle and 2-dtype0) or test_unaligned_layers_and_mixed_config'
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_kernels_gpu.py -m gpu -x -q -k "$SUBSET"
# hostile inputs: guard bands around unaligned views, non-finite buckets, full slices of 8/16/32/256-element
# buckets (lg 0/1/2/5), and a five-rank world
EDGE_SUBSET='w5- or (full_slices and (4-8 or 4-16 or 4-32 or 4-256 or 7-8 or 6-16)) or (standalone and f32-5- and (-8] or -32] or -1]))'
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_kernels_edge_gpu.py -m gpu -x -q -k "$EDGE_SUBSET"
# compressed reduce-scatter: edge inputs at W 2/3/5 (aligned, unaligned and aliased views), several windows, and
# interleaved reduce-scatter / allreduce / one-shot calls on one heap
RS_SUBSET='(edge_inputs and (w2-float32-q1- or w3-float16-q2- or w5-bfloat16-q3-)) or many_windows or interleaved'
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_reduce_scatter_gpu.py -m gpu -x -q -k "$RS_SUBSET"
# compressed all-gather: edge inputs at W 2/3/5 (separate and in-place inputs, unaligned views), several windows,
# and interleaved all-gather / reduce-scatter / allreduce / one-shot calls on one heap
AG_SUBSET='(edge_inputs and (w2-float32-q1- or w3-float16-q2- or w5-bfloat16-q3-)) or many_windows or interleaved'
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_all_gather_gpu.py -m gpu -x -q -k "$AG_SUBSET"
# all-to-all FP8 wire formats: edge inputs on unaligned views (full slices and bucket items), small slots with many
# windows, the routed form, FP8 / max-min / raw calls on one heap, and the generic reducer's FP8 item kernels
FP8_SUBSET='edge_inputs or small_slots or (routed and float32) or interleaved or (generic_path and float16)'
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_a2a_fp8_gpu.py -m gpu -x -q -k "$FP8_SUBSET"
# generic reducers on one GPU (quantize / accumulate / quantize_f32 / dequantize item kernels): SRA, Ring,
# all-to-all and the compressed broadcast at W = 3 on unaligned views, and the 1024-element slice path
RED_SUBSET='(match_host_and_reference and w3-float32-) or (width_and_slice_variants and 4-1024)'
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_reducers_local_gpu.py -m gpu -x -q -k "$RED_SUBSET"
# the allreduce engine with W engines on one GPU: fused groups halved and replayed from the bucket fast
# path, a two-level hierarchy with the compressed broadcast, the sharded collectives
ENG_SUBSET='(single_node and w2-float32) or (replays_the_slow_path and sr-2) or w4l2-SRA-RING or reduce_scatter_and_all_gather'
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_engine_local_gpu.py -m gpu -x -q -k "$ENG_SUBSET"
# the sharded collectives over several nodes: Reducer::reduce_scatter / all_gather through CudaBackend, the
# engine's two stages with and without heaps, the one-node NCCL-transport path
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_sharded_hierarchy_gpu.py -m gpu -x -q -k "not across_nodes"
# ResNet residual join: 16-byte and scalar paths, tails, unaligned views, with and without gb (the
# 103 M-element layer1 shapes and the training steps are left to the normal GPU run)
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_residual_relu_gpu.py -m gpu -x -q -k "not layer1 and not training_step"
# channels_last BatchNorm forward and backward: vector and one-element paths, single-block shapes, the
# grid merge (staging, self-resetting counters) on the one-element path with a partial last slab
# (8x100x16x16), unaligned views (the flagship shapes and the training steps are left to the normal GPU run)
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_batchnorm_gpu.py -m gpu -x -q -k "small_shapes or unaligned or rejects or fallbacks"
# the chain kernels' launch geometries (GY at 8 / 9 / 127, L = 1..13, partial slabs, graph capture), under
# memcheck and, since their chains, merges and trees meet in shared memory, under racecheck
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_batchnorm_mapping_gpu.py -m gpu -x -q
compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests/test_batchnorm_mapping_gpu.py -m gpu -x -q
# quantization-error estimator: 16-byte and scalar loads, bucket sizes 8..8192 and non-multiples of 8,
# tails, non-finite buckets, binding errors (the DDP run is left to the normal GPU run)
compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_adaptive_bits_gpu.py -m gpu -x -q -k "not ddp and not round_trip"
