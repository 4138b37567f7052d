"""The weight-gradient convolutions of one training step of R50-I3D-NL at 2 clips of 32 x 224^2 (the benchmarked network),
one entry per distinct geometry, with the number of its launches per step.  Shared by tests/gemm_paths.py (the
production cases of its table), tests/test_gpu_deterministic.py and scripts/bench_wgrad.py.

Entry: (label, in_shape (N, T, H, W, C), Co, kernel, strides, pads, dilations, launches per step).  conv1 has C = 4 (RGB
plus the zero pad channel the library's stem path expects)."""

PRODUCTION = [
    ('conv1 5x7x7 s2', (2, 32, 224, 224, 4), 64, (5, 7, 7), (1, 2, 2), (2, 3, 3), (1, 1, 1), 1),
    # res2: 56^2 x 32 frames, 3 blocks, a temporal 3x1x1 branch2a in every block
    ('res2_0_2a 3x1x1 64->64', (2, 32, 56, 56, 64), 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), 1),
    ('res2_x_2a 3x1x1 256->64', (2, 32, 56, 56, 256), 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), 2),
    ('res2_2b 1x3x3 64->64', (2, 32, 56, 56, 64), 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), 3),
    ('res2_2c/branch1 1x1 64->256', (2, 32, 56, 56, 64), 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 4),
    # res3: 16 frames after pool2; the first block strides 56^2 -> 28^2
    ('res3_0_2a 3x1x1 256->128', (2, 16, 56, 56, 256), 128, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), 1),
    ('res3_0_2b 1x3x3 s2 128->128', (2, 16, 56, 56, 128), 128, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), 1),
    ('res3_0_branch1 1x1 s2 256->512', (2, 16, 56, 56, 256), 512, (1, 1, 1), (1, 2, 2), (0, 0, 0), (1, 1, 1), 1),
    ('res3_2c 1x1 128->512', (2, 16, 28, 28, 128), 512, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 4),
    ('res3_x_2a 1x1 512->128', (2, 16, 28, 28, 512), 128, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 2),
    ('res3_2_2a 3x1x1 512->128', (2, 16, 28, 28, 512), 128, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), 1),
    ('res3_x_2b 1x3x3 128->128', (2, 16, 28, 28, 128), 128, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), 3),
    # res4: the first block strides 28^2 -> 14^2
    ('res4_0_2a 3x1x1 512->256', (2, 16, 28, 28, 512), 256, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), 1),
    ('res4_0_2b 1x3x3 s2 256->256', (2, 16, 28, 28, 256), 256, (1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 1, 1), 1),
    ('res4_0_branch1 1x1 s2 512->1024', (2, 16, 28, 28, 512), 1024, (1, 1, 1), (1, 2, 2), (0, 0, 0), (1, 1, 1), 1),
    ('res4_2c 1x1 256->1024', (2, 16, 14, 14, 256), 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 6),
    ('res4_x_2a 1x1 1024->256', (2, 16, 14, 14, 1024), 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 3),
    ('res4_x_2a 3x1x1 1024->256', (2, 16, 14, 14, 1024), 256, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), 2),
    ('res4_x_2b 1x3x3 256->256', (2, 16, 14, 14, 256), 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1), 5),
    # res5: stride 1, dilation 2 on the 3x3
    ('res5_0_2a 1x1 1024->512', (2, 16, 14, 14, 1024), 512, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 1),
    ('res5_0_branch1 1x1 1024->2048', (2, 16, 14, 14, 1024), 2048, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 1),
    ('res5_2b 1x3x3 d2 512->512', (2, 16, 14, 14, 512), 512, (1, 3, 3), (1, 1, 1), (0, 2, 2), (1, 2, 2), 3),
    ('res5_2c 1x1 512->2048', (2, 16, 14, 14, 512), 2048, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 3),
    ('res5_1_2a 3x1x1 2048->512', (2, 16, 14, 14, 2048), 512, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1), 1),
    ('res5_2_2a 1x1 2048->512', (2, 16, 14, 14, 2048), 512, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1), 1),
]


def out_dims(shape, ker, st, pd, dil):
    _, T, H, W, _ = shape
    return tuple((x + 2 * p - d * (k - 1) - 1) // s + 1 for x, k, s, p, d in zip((T, H, W), ker, st, pd, dil))


def useful_flops(shape, co, ker, st, pd, dil):
    """2 x positions x Co x taps x real input channels (conv1: 3 colour channels, 7 columns)."""
    To, Ho, Wo = out_dims(shape, ker, st, pd, dil)
    ci = 3 if shape[4] == 4 else shape[4]
    return 2.0 * shape[0] * To * Ho * Wo * co * ker[0] * ker[1] * ker[2] * ci


def min_bytes(shape, co, ker, st, pd, dil):
    """dY and X read once, dw read and written once (fp32)."""
    To, Ho, Wo = out_dims(shape, ker, st, pd, dil)
    n, t, h, w, c = shape
    dw = co * ker[0] * ker[1] * (8 if c == 4 else ker[2]) * c
    return 4.0 * (n * To * Ho * Wo * co + n * t * h * w * c + 2 * dw)
