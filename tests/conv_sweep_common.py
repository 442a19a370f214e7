"""The covering parity sweep of the tensor-core convolution engine: the case table and the coverage classes.

Every case is one convolution run through danet_conv_tc_group on the GPU (tests/test_conv_sweep_gpu.py) against an fp64
reference.  Which tile body, swizzle, tap grouping, K segments, stacking and pairing form a case exercises is not
visible in its shape; danet_conv_tc_dispatch reports it from the engine's own make_prob, and CLASSES states, as
predicates over that report and the case fields, everything the table has to cover.  tests/test_conv_sweep_cpu.py fails
with the names of the uncovered classes, so a change to make_prob (a new tile width, another stacking rule) shows up
without a GPU.

Combinations make_prob cannot produce, and which therefore have no class: several channel chunks at 32- or 64-byte
swizzle (those widths are chosen only for Cin <= 32, one chunk), and a last chunk with fewer K steps than a full one
at those widths (a chunk is one or two K steps and Cin fills all but the last 8 channels of them)."""
import ctypes

import fp64_bound as fb

# N, H, W, Cin, Cout, k, stride, wsets, relu, residual (none | f32 | planes), output (f32 | planes | both), bias, precision
CASES = [
    (2, 12, 10, 16, 16, 1, 1, 1, 0, "none", "f32", 0, "fast"),  # fast NT 16 full
    (3, 13, 9, 8, 8, 1, 2, 1, 1, "none", "both", 0, "fast"),  # fast NT 16 ragged
    (1, 20, 12, 24, 32, 3, 1, 1, 0, "f32", "planes", 1, "fast"),  # fast NT 32 full
    (2, 17, 11, 32, 24, 3, 1, 1, 1, "planes", "f32", 1, "fast"),  # fast NT 32 ragged
    (3, 22, 18, 40, 48, 3, 2, 1, 0, "planes", "planes", 0, "fast"),  # fast NT 48 full
    (1, 21, 15, 64, 40, 3, 2, 1, 1, "none", "f32", 0, "fast"),  # fast NT 48 ragged
    (2, 36, 20, 8, 64, 7, 2, 1, 0, "none", "both", 1, "fast"),  # fast NT 64 full
    (3, 35, 19, 24, 56, 7, 2, 1, 1, "f32", "planes", 1, "fast"),  # fast NT 64 ragged
    (1, 10, 20, 128, 80, 1, 1, 1, 0, "f32", "both", 0, "fast"),  # fast NT 80 full
    (2, 9, 7, 72, 72, 1, 2, 1, 1, "planes", "planes", 0, "fast"),  # fast NT 80 ragged
    (3, 18, 12, 104, 96, 3, 1, 1, 0, "none", "f32", 1, "fast"),  # fast NT 96 full
    (1, 11, 13, 192, 88, 1, 2, 1, 1, "none", "both", 1, "fast"),  # fast NT 96 ragged
    (2, 12, 10, 16, 112, 1, 1, 1, 0, "f32", "f32", 0, "fast"),  # fast NT 112 full
    (3, 13, 9, 8, 104, 1, 2, 1, 1, "f32", "both", 0, "fast"),  # fast NT 112 ragged
    (1, 20, 12, 24, 128, 3, 1, 1, 0, "planes", "planes", 1, "fast"),  # fast NT 128 full
    (2, 17, 11, 32, 120, 3, 1, 1, 1, "none", "f32", 1, "fast"),  # fast NT 128 ragged
    (3, 22, 18, 40, 144, 3, 2, 1, 0, "none", "planes", 0, "fast"),  # fast NT 144 full
    (1, 21, 15, 64, 136, 3, 2, 1, 1, "f32", "f32", 0, "fast"),  # fast NT 144 ragged
    (2, 36, 20, 8, 160, 7, 2, 1, 0, "f32", "both", 1, "fast"),  # fast NT 160 full
    (3, 35, 19, 24, 152, 7, 2, 1, 1, "planes", "planes", 1, "fast"),  # fast NT 160 ragged
    (1, 10, 20, 128, 176, 1, 1, 1, 0, "planes", "both", 0, "fast"),  # fast NT 176 full
    (2, 9, 7, 72, 168, 1, 2, 1, 1, "none", "planes", 0, "fast"),  # fast NT 176 ragged
    (3, 18, 12, 104, 192, 3, 1, 1, 0, "f32", "f32", 1, "fast"),  # fast NT 192 full
    (1, 11, 13, 192, 184, 1, 2, 1, 1, "f32", "both", 1, "fast"),  # fast NT 192 ragged
    (2, 12, 10, 16, 208, 1, 1, 1, 0, "planes", "f32", 0, "fast"),  # fast NT 208 full
    (3, 13, 9, 8, 200, 1, 2, 1, 1, "planes", "both", 0, "fast"),  # fast NT 208 ragged
    (1, 20, 12, 24, 224, 3, 1, 1, 0, "none", "planes", 1, "fast"),  # fast NT 224 full
    (2, 17, 11, 32, 216, 3, 1, 1, 1, "f32", "f32", 1, "fast"),  # fast NT 224 ragged
    (3, 22, 18, 40, 240, 3, 2, 1, 0, "f32", "planes", 0, "fast"),  # fast NT 240 full
    (1, 21, 15, 64, 232, 3, 2, 1, 1, "planes", "f32", 0, "fast"),  # fast NT 240 ragged
    (2, 36, 20, 8, 256, 7, 2, 1, 0, "planes", "both", 1, "fast"),  # fast NT 256 full
    (3, 35, 19, 24, 248, 7, 2, 1, 1, "none", "planes", 1, "fast"),  # fast NT 256 ragged
    (2, 14, 10, 48, 272, 3, 1, 1, 0, "none", "both", 0, "fast"),  # fast, 2 N tiles of 144, ragged last
    (1, 9, 12, 32, 520, 1, 1, 1, 1, "f32", "planes", 0, "fast"),  # fast, 3 N tiles of 176, ragged last
    (2, 8, 8, 64, 512, 1, 1, 1, 0, "planes", "f32", 1, "fast"),  # fast, 2 full N tiles
    (2, 12, 10, 16, 16, 1, 1, 1, 0, "none", "f32", 0, "exact"),  # exact Cout 16
    (3, 13, 9, 8, 16, 1, 2, 1, 1, "none", "both", 0, "exact"),  # exact Cout 16
    (1, 20, 12, 24, 8, 3, 1, 1, 0, "f32", "planes", 1, "exact"),  # exact Cout 8
    (2, 17, 11, 32, 8, 3, 1, 1, 1, "planes", "f32", 1, "exact"),  # exact Cout 8
    (3, 22, 18, 40, 32, 3, 2, 1, 0, "planes", "planes", 0, "exact"),  # exact Cout 32
    (1, 21, 15, 64, 32, 3, 2, 1, 1, "none", "f32", 0, "exact"),  # exact Cout 32
    (2, 36, 20, 8, 24, 7, 2, 1, 0, "none", "both", 1, "exact"),  # exact Cout 24
    (3, 35, 19, 24, 24, 7, 2, 1, 1, "f32", "planes", 1, "exact"),  # exact Cout 24
    (1, 10, 20, 128, 48, 1, 1, 1, 0, "f32", "both", 0, "exact"),  # exact Cout 48
    (2, 9, 7, 72, 48, 1, 2, 1, 1, "planes", "planes", 0, "exact"),  # exact Cout 48
    (3, 18, 12, 104, 40, 3, 1, 1, 0, "none", "f32", 1, "exact"),  # exact Cout 40
    (1, 11, 13, 192, 40, 1, 2, 1, 1, "none", "both", 1, "exact"),  # exact Cout 40
    (2, 12, 10, 16, 64, 1, 1, 1, 0, "f32", "f32", 0, "exact"),  # exact Cout 64
    (3, 13, 9, 8, 64, 1, 2, 1, 1, "f32", "both", 0, "exact"),  # exact Cout 64
    (1, 20, 12, 24, 56, 3, 1, 1, 0, "planes", "planes", 1, "exact"),  # exact Cout 56
    (2, 17, 11, 32, 56, 3, 1, 1, 1, "none", "f32", 1, "exact"),  # exact Cout 56
    (3, 22, 18, 40, 96, 3, 2, 1, 0, "none", "planes", 0, "exact"),  # exact Cout 96
    (1, 21, 15, 64, 96, 3, 2, 1, 1, "f32", "f32", 0, "exact"),  # exact Cout 96
    (2, 36, 20, 8, 72, 7, 2, 1, 0, "f32", "both", 1, "exact"),  # exact Cout 72
    (3, 35, 19, 24, 72, 7, 2, 1, 1, "planes", "planes", 1, "exact"),  # exact Cout 72
    (1, 10, 20, 128, 192, 1, 1, 1, 0, "planes", "both", 0, "exact"),  # exact Cout 192
    (2, 9, 7, 72, 192, 1, 2, 1, 1, "none", "planes", 0, "exact"),  # exact Cout 192
    (3, 18, 12, 104, 136, 3, 1, 1, 0, "f32", "f32", 1, "exact"),  # exact Cout 136
    (1, 11, 13, 192, 136, 1, 2, 1, 1, "f32", "both", 1, "exact"),  # exact Cout 136
    (3, 1, 20, 48, 32, 3, 1, 1, 0, "planes", "f32", 0, "exact"),  # H = 1, exact
    (3, 1, 20, 48, 32, 3, 1, 1, 1, "planes", "both", 1, "fast"),  # H = 1, fast
    (3, 20, 1, 48, 32, 3, 1, 1, 1, "planes", "both", 0, "exact"),  # W = 1, exact
    (3, 20, 1, 48, 32, 3, 1, 1, 0, "none", "f32", 0, "fast"),  # W = 1, fast
    (2, 1, 9, 16, 16, 3, 2, 1, 0, "none", "planes", 1, "exact"),  # H = 1, stride 2, exact
    (2, 1, 9, 16, 16, 3, 2, 1, 1, "none", "both", 0, "fast"),  # H = 1, stride 2, fast
    (2, 33, 1, 16, 24, 7, 2, 1, 1, "f32", "f32", 1, "exact"),  # W = 1, 7x7, exact
    (2, 33, 1, 16, 24, 7, 2, 1, 0, "f32", "planes", 1, "fast"),  # W = 1, 7x7, fast
    (5, 1, 1, 64, 64, 1, 1, 1, 0, "f32", "planes", 0, "exact"),  # 1x1 map, exact
    (5, 1, 1, 64, 64, 1, 1, 1, 1, "planes", "f32", 1, "fast"),  # 1x1 map, fast
    (1, 40, 5, 32, 48, 3, 1, 1, 1, "planes", "f32", 0, "exact"),  # Wo < 8, tall, exact
    (1, 40, 5, 32, 48, 3, 1, 1, 0, "planes", "planes", 0, "fast"),  # Wo < 8, tall, fast
    (1, 56, 24, 64, 64, 3, 1, 1, 0, "planes", "both", 1, "exact"),  # 4 tile rows, exact
    (1, 56, 24, 64, 64, 3, 1, 1, 1, "none", "f32", 0, "fast"),  # 4 tile rows, fast
    (1, 40, 16, 64, 64, 3, 1, 1, 1, "none", "planes", 1, "exact"),  # 3 tile rows, exact
    (1, 40, 16, 64, 64, 3, 1, 1, 0, "none", "both", 1, "fast"),  # 3 tile rows, fast
    (1, 56, 56, 64, 64, 7, 2, 1, 0, "none", "both", 0, "exact"),  # 7x7/s2 stem, 2 tile rows, exact
    (1, 56, 56, 64, 64, 7, 2, 1, 1, "f32", "planes", 1, "fast"),  # 7x7/s2 stem, 2 tile rows, fast
    (1, 70, 9, 16, 16, 1, 1, 1, 1, "f32", "planes", 0, "exact"),  # 5 tile rows, 1x1, exact
    (1, 70, 9, 16, 16, 1, 1, 1, 0, "f32", "both", 0, "fast"),  # 5 tile rows, 1x1, fast
    (4, 14, 14, 64, 96, 3, 1, 1, 0, "planes", "f32", 1, "exact"),  # one tile row, 4 images, exact
    (4, 14, 14, 64, 96, 3, 1, 1, 1, "planes", "planes", 0, "fast"),  # one tile row, 4 images, fast
    (5, 14, 14, 64, 96, 3, 1, 1, 1, "planes", "both", 1, "exact"),  # one tile row, 5 images, exact
    (5, 14, 14, 64, 96, 3, 1, 1, 0, "none", "f32", 1, "fast"),  # one tile row, 5 images, fast
    (1, 16, 8, 128, 64, 3, 1, 1, 0, "none", "f32", 0, "exact"),  # one tile row, N = 1, exact
    (1, 16, 8, 128, 64, 3, 1, 1, 1, "none", "both", 1, "fast"),  # one tile row, N = 1, fast
    (5, 7, 7, 64, 64, 3, 1, 1, 1, "none", "both", 0, "exact"),  # 7x7 maps: 2 per tile, ragged count, exact
    (5, 7, 7, 64, 64, 3, 1, 1, 0, "f32", "f32", 0, "fast"),  # 7x7 maps: 2 per tile, ragged count, fast
    (7, 4, 4, 128, 64, 3, 1, 1, 0, "f32", "planes", 1, "exact"),  # 4x4 maps: 3 per tile, exact
    (7, 4, 4, 128, 64, 3, 1, 1, 1, "f32", "both", 0, "fast"),  # 4x4 maps: 3 per tile, fast
    (9, 3, 3, 40, 32, 3, 1, 1, 1, "planes", "f32", 1, "exact"),  # 3x3 maps: 4 per tile, exact
    (9, 3, 3, 40, 32, 3, 1, 1, 0, "planes", "planes", 1, "fast"),  # 3x3 maps: 4 per tile, fast
    (11, 2, 2, 512, 64, 3, 1, 1, 0, "planes", "planes", 0, "exact"),  # 2x2 maps: 5 per tile, exact
    (11, 2, 2, 512, 64, 3, 1, 1, 1, "none", "f32", 1, "fast"),  # 2x2 maps: 5 per tile, fast
    (13, 1, 1, 64, 48, 3, 1, 1, 1, "none", "f32", 0, "exact"),  # 1x1 maps, 3x3 filter: 8 per tile, exact
    (13, 1, 1, 64, 48, 3, 1, 1, 0, "none", "planes", 0, "fast"),  # 1x1 maps, 3x3 filter: 8 per tile, fast
    (35, 1, 1, 2048, 32, 1, 1, 1, 0, "none", "both", 1, "exact"),  # 1x1 maps, 1x1 filter: 16 per tile, exact
    (35, 1, 1, 2048, 32, 1, 1, 1, 1, "f32", "f32", 0, "fast"),  # 1x1 maps, 1x1 filter: 16 per tile, fast
    (9, 4, 4, 32, 32, 1, 1, 1, 1, "f32", "planes", 1, "exact"),  # 4x4 maps, 1x1: 4 per tile, no zero rows, exact
    (9, 4, 4, 32, 32, 1, 1, 1, 0, "f32", "both", 1, "fast"),  # 4x4 maps, 1x1: 4 per tile, no zero rows, fast
    (2, 2, 2, 32, 48, 3, 1, 1, 0, "f32", "both", 0, "exact"),  # N < nstack, exact
    (2, 2, 2, 32, 48, 3, 1, 1, 1, "planes", "planes", 1, "fast"),  # N < nstack, fast
    (3, 1, 8, 16, 16, 1, 1, 1, 1, "planes", "planes", 0, "exact"),  # N < nstack, 16 per tile, exact
    (3, 1, 8, 16, 16, 1, 1, 1, 0, "planes", "both", 0, "fast"),  # N < nstack, 16 per tile, fast
    (5, 13, 13, 64, 64, 3, 2, 1, 0, "none", "f32", 1, "exact"),  # stride 2, 13x13 -> 7x7: 2 per tile, exact
    (5, 13, 13, 64, 64, 3, 2, 1, 1, "none", "planes", 0, "fast"),  # stride 2, 13x13 -> 7x7: 2 per tile, fast
    (7, 7, 7, 128, 64, 3, 2, 1, 1, "none", "both", 1, "exact"),  # stride 2, 7x7 -> 4x4: 3 per tile, exact
    (7, 7, 7, 128, 64, 3, 2, 1, 0, "f32", "f32", 1, "fast"),  # stride 2, 7x7 -> 4x4: 3 per tile, fast
    (6, 6, 6, 48, 32, 3, 2, 1, 0, "f32", "f32", 0, "exact"),  # stride 2, 6x6 -> 3x3: 4 per tile, exact
    (6, 6, 6, 48, 32, 3, 2, 1, 1, "f32", "both", 1, "fast"),  # stride 2, 6x6 -> 3x3: 4 per tile, fast
    (4, 4, 4, 256, 128, 3, 2, 1, 1, "f32", "both", 0, "exact"),  # stride 2, 4x4 -> 2x2: 5 per tile, exact
    (4, 4, 4, 256, 128, 3, 2, 1, 0, "planes", "f32", 0, "fast"),  # stride 2, 4x4 -> 2x2: 5 per tile, fast
    (17, 2, 2, 64, 32, 3, 2, 1, 0, "planes", "planes", 1, "exact"),  # stride 2, 2x2 -> 1x1: 8 per tile, exact
    (17, 2, 2, 64, 32, 3, 2, 1, 1, "planes", "both", 0, "fast"),  # stride 2, 2x2 -> 1x1: 8 per tile, fast
    (20, 2, 2, 64, 32, 1, 2, 1, 1, "none", "f32", 1, "exact"),  # 1x1/s2, 2x2 -> 1x1: 16 per tile, exact
    (20, 2, 2, 64, 32, 1, 2, 1, 0, "none", "planes", 1, "fast"),  # 1x1/s2, 2x2 -> 1x1: 16 per tile, fast
    (3, 8, 8, 24, 16, 1, 2, 1, 0, "none", "planes", 0, "exact"),  # 1x1/s2 on 8x8: 4 per tile, exact
    (3, 8, 8, 24, 16, 1, 2, 1, 1, "f32", "f32", 1, "fast"),  # 1x1/s2 on 8x8: 4 per tile, fast
    (264, 2, 2, 32, 48, 3, 1, 24, 1, "f32", "f32", 0, "exact"),  # 24 sets, 11 images per set: 5 + 5 + 1, exact
    (264, 2, 2, 32, 48, 3, 1, 24, 0, "f32", "planes", 0, "fast"),  # 24 sets, 11 images per set: 5 + 5 + 1, fast
    (24, 2, 2, 128, 128, 3, 1, 24, 0, "f32", "both", 1, "exact"),  # 24 sets, one image per set, exact
    (24, 2, 2, 128, 128, 3, 1, 24, 1, "planes", "f32", 0, "fast"),  # 24 sets, one image per set, fast
    (72, 4, 4, 64, 32, 3, 2, 24, 1, "planes", "planes", 1, "exact"),  # 24 sets, stacked stride 2, 3 per set, exact
    (72, 4, 4, 64, 32, 3, 2, 24, 0, "planes", "both", 1, "fast"),  # 24 sets, stacked stride 2, 3 per set, fast
    (24, 4, 4, 64, 32, 1, 2, 24, 0, "planes", "both", 0, "exact"),  # 24 sets, one image per set, stride 2, exact
    (24, 4, 4, 64, 32, 1, 2, 24, 1, "none", "planes", 1, "fast"),  # 24 sets, one image per set, stride 2, fast
    (24, 28, 12, 48, 24, 3, 1, 24, 1, "none", "planes", 0, "exact"),  # 24 sets on tall maps, exact
    (24, 28, 12, 48, 24, 3, 1, 24, 0, "none", "both", 0, "fast"),  # 24 sets on tall maps, fast
    (48, 10, 8, 16, 24, 3, 1, 24, 0, "f32", "f32", 1, "exact"),  # 24 sets, one-row maps, 2 per set, exact
    (48, 10, 8, 16, 24, 3, 1, 24, 1, "f32", "planes", 0, "fast"),  # 24 sets, one-row maps, 2 per set, fast
    (2, 7, 7, 384, 64, 3, 1, 1, 1, "f32", "both", 1, "exact"),  # 3x3x384, exact
    (2, 7, 7, 384, 64, 3, 1, 1, 0, "planes", "f32", 1, "fast"),  # 3x3x384, fast
    (2, 8, 8, 2048, 16, 1, 1, 1, 0, "planes", "f32", 0, "exact"),  # 1x1x2048 one block per chunk, exact
    (2, 8, 8, 2048, 16, 1, 1, 1, 1, "planes", "both", 1, "fast"),  # 1x1x2048 one block per chunk, fast
    (2, 16, 8, 16, 16, 1, 1, 1, 1, "planes", "both", 0, "exact"),  # a single K step, exact
    (2, 16, 8, 16, 16, 1, 1, 1, 0, "none", "f32", 0, "fast"),  # a single K step, fast
    (2, 20, 12, 64, 16, 7, 2, 1, 0, "none", "planes", 1, "exact"),  # 7x7/s2, narrow tile: 6-tap blocks, exact
    (2, 20, 12, 64, 16, 7, 2, 1, 1, "none", "both", 0, "fast"),  # 7x7/s2, narrow tile: 6-tap blocks, fast
    (2, 20, 12, 32, 16, 7, 2, 1, 1, "f32", "f32", 1, "exact"),  # 7x7/s2, 64-byte rows: 12-tap blocks, exact
    (2, 20, 12, 32, 16, 7, 2, 1, 0, "f32", "planes", 1, "fast"),  # 7x7/s2, 64-byte rows: 12-tap blocks, fast
    (2, 12, 8, 48, 16, 3, 1, 1, 0, "f32", "planes", 0, "exact"),  # 3x3, 3 K steps: 18 + 9, exact
    (2, 12, 8, 48, 16, 3, 1, 1, 1, "planes", "f32", 1, "fast"),  # 3x3, 3 K steps: 18 + 9, fast
    (2, 9, 13, 192, 16, 1, 1, 1, 1, "planes", "f32", 0, "exact"),  # 1x1 on an odd map, 3 chunks, exact
    (2, 9, 13, 192, 16, 1, 1, 1, 0, "planes", "planes", 0, "fast"),  # 1x1 on an odd map, 3 chunks, fast
]

FIELDS = ("NT", "ntn", "last_nt", "SWB", "KCH", "nchunks", "kv_last", "npa", "ntap", "TG", "ngrp", "nstack", "hs",
          "tiles_h", "tiles_w", "nblk", "closes", "longest", "closes_plane_end", "closes_mid_plane", "pairing", "pairs",
          "pairs_past")
EXACT_FLAG = 4
# the longest K segment make_prob can produce (main-chain MMAs), over the shape grid test_conv_sweep_cpu.py enumerates
LONGEST_SEGMENT = 24


def base(case):
    """the 10-field case of conv_tc_common (residual as a flag)"""
    return tuple(case[:9]) + (int(case[9] != "none"),)


def out_hw(case):
    N, H, W, Cin, Cout, k, s = case[:7]
    return (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1


def dispatch(N, H, W, Cin, Cout, k, s, G, exact, pad=None):
    """danet_conv_tc_dispatch as a dict, or None if the engine does not take the shape.  Host only."""
    from danet_b200 import _lib as L
    d = L.ConvDesc(N, H, W, Cin, Cout, k, s, k // 2 if pad is None else pad, G, 0, EXACT_FLAG if exact else 0)
    out = (ctypes.c_int64 * len(FIELDS))()
    if L.load().danet_conv_tc_dispatch(ctypes.byref(d), ctypes.cast(out, ctypes.c_void_p)) != 0:
        return None
    return dict(zip(FIELDS, list(out)))


def report(case):
    r = dispatch(*case[:8], exact=case[12] == "exact")
    assert r is not None, ("the engine does not take this case", case)
    return r


def _classes():
    """[(name, predicate((case, report)))]"""
    cl = []

    def add(name, fn):
        cl.append((name, lambda cr: fn(*cr)))

    def prec(p):
        return lambda c: c[12] == p

    for p, widths in (("exact", range(16, 65, 16)), ("fast", range(16, 257, 16))):
        is_p = prec(p)
        for nt in widths:
            add("%s NT %d, full last N tile" % (p, nt), lambda c, r, is_p=is_p, nt=nt: is_p(c) and r["NT"] == nt and r["last_nt"] == nt)
            add("%s NT %d, ragged last N tile" % (p, nt), lambda c, r, is_p=is_p, nt=nt: is_p(c) and r["NT"] == nt and r["last_nt"] < nt)
        add("%s Cout %% 16 == 8" % p, lambda c, r, is_p=is_p: is_p(c) and c[4] % 16 == 8)
        add("%s one N tile" % p, lambda c, r, is_p=is_p: is_p(c) and r["ntn"] == 1)
        add("%s two N tiles" % p, lambda c, r, is_p=is_p: is_p(c) and r["ntn"] == 2)
        add("%s three or more N tiles" % p, lambda c, r, is_p=is_p: is_p(c) and r["ntn"] >= 3)
        add("%s three or more N tiles, ragged last" % p, lambda c, r, is_p=is_p: is_p(c) and r["ntn"] >= 3 and r["last_nt"] < r["NT"])
        # swizzle width x channel chunks
        for swb in (32, 64):
            add("%s SWB %d, Cin fills the chunk" % (p, swb), lambda c, r, is_p=is_p, swb=swb: is_p(c) and r["SWB"] == swb and c[3] == r["KCH"])
            add("%s SWB %d, Cin short of the chunk" % (p, swb), lambda c, r, is_p=is_p, swb=swb: is_p(c) and r["SWB"] == swb and c[3] < r["KCH"])
        add("%s SWB 128, one full chunk" % p, lambda c, r, is_p=is_p: is_p(c) and r["SWB"] == 128 and r["nchunks"] == 1 and r["kv_last"] == 4)
        add("%s SWB 128, one chunk of fewer K steps" % p, lambda c, r, is_p=is_p: is_p(c) and r["SWB"] == 128 and r["nchunks"] == 1 and r["kv_last"] < 4)
        add("%s SWB 128, several full chunks" % p, lambda c, r, is_p=is_p: is_p(c) and r["SWB"] == 128 and r["nchunks"] > 1 and c[3] % 64 == 0)
        add("%s SWB 128, several chunks, last of fewer K steps" % p,
            lambda c, r, is_p=is_p: is_p(c) and r["SWB"] == 128 and r["nchunks"] > 1 and r["kv_last"] < 4)
        add("%s last K step half filled (Cin %% 16 == 8), several chunks" % p,
            lambda c, r, is_p=is_p: is_p(c) and r["nchunks"] > 1 and c[3] % 16 == 8)
        # filter x stride x map parity, and degenerate maps
        for k, s in ((1, 1), (1, 2), (3, 1), (3, 2), (7, 2)):
            for name, idx, par in (("even H", 1, 0), ("odd H", 1, 1), ("even W", 2, 0), ("odd W", 2, 1)):
                add("%s %dx%d/s%d, %s" % (p, k, k, s, name),
                    lambda c, r, is_p=is_p, k=k, s=s, idx=idx, par=par: is_p(c) and c[5] == k and c[6] == s and c[idx] % 2 == par and c[idx] > 1)
        add("%s H = 1" % p, lambda c, r, is_p=is_p: is_p(c) and c[1] == 1 and c[2] > 1)
        add("%s W = 1" % p, lambda c, r, is_p=is_p: is_p(c) and c[2] == 1 and c[1] > 1)
        add("%s Wo < 8 on a map of several tile rows" % p, lambda c, r, is_p=is_p: is_p(c) and out_hw(c)[1] < 8 and r["tiles_h"] > 1)
        add("%s Ho %% 16 != 0, several tile rows" % p, lambda c, r, is_p=is_p: is_p(c) and out_hw(c)[0] % 16 != 0 and r["tiles_h"] > 1)
        add("%s Wo %% 8 != 0, several tile columns" % p, lambda c, r, is_p=is_p: is_p(c) and out_hw(c)[1] % 8 != 0 and r["tiles_w"] > 1)
        # tap groups
        add("%s one weight block per parity plane (TG == taps), several taps" % p, lambda c, r, is_p=is_p: is_p(c) and r["ntap"] > 1 and r["TG"] == r["ntap"])
        add("%s several weight blocks per parity plane (TG < taps)" % p, lambda c, r, is_p=is_p: is_p(c) and 1 < r["TG"] < r["ntap"])
        add("%s one tap per weight block" % p, lambda c, r, is_p=is_p: is_p(c) and r["TG"] == 1 and r["ntap"] > 1)
        add("%s last weight block of a plane holds fewer taps" % p, lambda c, r, is_p=is_p: is_p(c) and r["TG"] > 1 and r["ntap"] % r["TG"] != 0 and r["ntap"] > r["TG"])
        # stacking
        for ns in (2, 3, 4, 5, 8, 16):
            add("%s %d images per tile" % (p, ns), lambda c, r, is_p=is_p, ns=ns: is_p(c) and r["nstack"] == ns)
        for s in (1, 2):
            add("%s stacked, stride %d" % (p, s), lambda c, r, is_p=is_p, s=s: is_p(c) and r["nstack"] > 1 and c[6] == s)
            add("%s stacked, stride %d, 24 weight sets" % (p, s), lambda c, r, is_p=is_p, s=s: is_p(c) and r["nstack"] > 1 and c[6] == s and c[7] == 24)
        add("%s stacked, ragged image count" % p, lambda c, r, is_p=is_p: is_p(c) and r["nstack"] > 1 and c[7] == 1 and c[0] % r["nstack"] != 0 and c[0] > r["nstack"])
        add("%s stacked, N < images per tile" % p, lambda c, r, is_p=is_p: is_p(c) and c[7] == 1 and c[0] < r["nstack"])
        add("%s stacked, 24 weight sets, ragged images per set" % p,
            lambda c, r, is_p=is_p: is_p(c) and r["nstack"] > 1 and c[7] == 24 and (c[0] // 24) % r["nstack"] != 0 and c[0] // 24 > r["nstack"])
        add("%s stacked, 24 weight sets, one image per set" % p, lambda c, r, is_p=is_p: is_p(c) and r["nstack"] > 1 and c[7] == 24 and c[0] == 24)
        add("%s 24 weight sets, one image per tile" % p, lambda c, r, is_p=is_p: is_p(c) and r["nstack"] == 1 and c[7] == 24)
        add("%s N = 1" % p, lambda c, r, is_p=is_p: is_p(c) and c[0] == 1)
        # residual x output x bias x relu, pairwise
        kinds = (("residual", 9, ("none", "f32", "planes")), ("output", 10, ("f32", "planes", "both")), ("bias", 11, (0, 1)), ("relu", 8, (0, 1)))
        for a in range(len(kinds)):
            for b in range(a + 1, len(kinds)):
                for va in kinds[a][2]:
                    for vb in kinds[b][2]:
                        add("%s %s %s x %s %s" % (p, kinds[a][0], va, kinds[b][0], vb),
                            lambda c, r, is_p=is_p, ia=kinds[a][1], ib=kinds[b][1], va=va, vb=vb: is_p(c) and c[ia] == va and c[ib] == vb)
    # exact mode only: K segments and tile pairs
    ex = prec("exact")
    add("exact one K segment", lambda c, r: ex(c) and r["closes"] == 1)
    add("exact several K segments", lambda c, r: ex(c) and r["closes"] >= 3)
    add("exact K segment closes at a parity plane's end before the last plane", lambda c, r: ex(c) and r["closes_plane_end"] > 0)
    add("exact K segment closes inside a parity plane", lambda c, r: ex(c) and r["closes_mid_plane"] > 0)
    add("exact K segment spans a parity plane's end", lambda c, r: ex(c) and r["closes"] < r["nblk"] and r["npa"] * r["nchunks"] > 1
        and r["closes_mid_plane"] + r["closes_plane_end"] + 1 < r["npa"] * r["nchunks"])
    add("exact longest K segment the engine produces", lambda c, r: ex(c) and r["longest"] == LONGEST_SEGMENT)
    add("exact row pairs, even tile rows", lambda c, r: ex(c) and r["pairing"] == 1 and r["tiles_h"] % 2 == 0)
    add("exact row pairs, odd tile rows", lambda c, r: ex(c) and r["pairing"] == 1 and r["tiles_h"] % 2 == 1 and r["pairs_past"] > 0)
    add("exact image-group pairs, every pair complete", lambda c, r: ex(c) and r["pairing"] == 2 and r["pairs"] > 0 and r["pairs_past"] == 0)
    add("exact image-group pairs, a second tile past the images", lambda c, r: ex(c) and r["pairing"] == 2 and r["pairs_past"] > 0 and r["pairs"] > r["pairs_past"])
    add("exact image-group pairs, no pair complete", lambda c, r: ex(c) and r["pairing"] == 2 and r["pairs"] == r["pairs_past"])
    add("exact image-group pairs, 24 weight sets", lambda c, r: ex(c) and r["pairing"] == 2 and c[7] == 24 and r["pairs"] > r["pairs_past"])
    add("exact row pairs, 24 weight sets", lambda c, r: ex(c) and r["pairing"] == 1 and c[7] == 24)
    return cl


CLASSES = _classes()


def coverage(cases=None):
    """{class name: [indices of the cases in it]}"""
    cases = CASES if cases is None else cases
    return fb.coverage([(c, report(c)) for c in cases], CLASSES)
