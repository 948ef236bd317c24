"""The cases of tests/test_gpu_smt_cnn_domain.py as plain data, shared with tests/test_smt_cnn_domain_host.py, which
checks that they reach every bin shape, crop origin, resize limit, stem K split and head layout ``ssb_smt_cnn_batch``
accepts.

An input is a dict: an H x W observation with C channels, read with ``scale`` 1 (RGB: x / 255) or 0 (depth), resized
to rh x rw and cropped at (cy, cx), into a network whose fc has ``n_out`` outputs and a bias when ``bias``.  A case is
one call: one or two inputs (RGB first) and a batch size.
"""
from smt_cnn_models import geometry

CHANNELS = (1, 2, 3, 4, 5, 8)


def modality(H, W, C, scale, n_out=64, bias=True, geom=None):
    rh, rw, cy, cx = geom or geometry(H, W)
    return dict(H=H, W=W, C=C, scale=scale, rh=rh, rw=rw, cy=cy, cx=cx, n_out=n_out, bias=bias)


def case(name, *inputs, B=2):
    return dict(name=name, inputs=list(inputs), B=B)


# Shapes through the reference's own geometry.  Bin widths (rows / columns): 1 x 1 and 2 x 2 inputs every bin 1 wide;
# 3 - 63 and 17 x 900 upsample with 1- and 2-wide bins that share a pixel; 65 and 65 x 1000: 2; 127: 2 / 3; 129: 3;
# 255: 4 / 5; 341 x 256: 5 rows by 4 columns, rows 0 - 39 and 297 - 340 never read; 480 x 640 and 640 x 480: 8 by
# 8 / 9, crop 10 off the long axis; 1000 and 1023: 16 / 17; 1024: exactly 16.  1024 x 64 and 64 x 1024 crop 64 of 1024
# rows or columns at 480; 1 x 1024 and 1024 x 1 resize to 65536 (the entry's limit) and read 2 of the 1024 at 32736;
# 2 x 1023 resizes to 32736.  The short edges that round to 63 (49, 98, ...) are refused and tested elsewhere.
SQUARES = (1, 2, 3, 7, 31, 33, 63, 65, 127, 129, 255, 1000, 1023, 1024)
OBLONG = ((480, 640), (640, 480), (1024, 64), (64, 1024), (341, 256), (1, 1024), (1024, 1), (2, 1023), (17, 900),
          (65, 1000))
SHAPES = [(m, m) for m in SQUARES] + list(OBLONG)

# every shape runs RGB and depth together, their channels stepping through CHANNELS at different offsets, so each C
# meets both scales several times and network 0 has the larger K split in some calls and the smaller in others
SHAPE_CASES = [case(f"s{H}x{W}", modality(H, W, CHANNELS[i % 6], 1), modality(H, W, CHANNELS[(i + 2) % 6], 0))
               for i, (H, W) in enumerate(SHAPES)]

# two inputs of different geometries and heads in one call: the column offset of input 1 and the row stride
PAIR_CASES = [
    # S = 1 (C = 2, K = 98) before S = 4 (C = 8); n_out 257 then 1
    case("pair_s1_s4_257_1", modality(130, 70, 2, 1, n_out=257), modality(33, 33, 8, 0, n_out=1), B=3),
    # S = 4 (C = 5) before S = 1 (C = 1); RGB's fc without a bias, n_out 100 then 64
    case("pair_s4_s1_nobias", modality(96, 128, 5, 1, n_out=100, bias=False), modality(640, 480, 1, 0), B=3),
    # equal C at different geometries; depth's fc without a bias
    case("pair_equal_c", modality(255, 255, 3, 1, n_out=1), modality(48, 48, 3, 0, n_out=257, bias=False), B=3),
    # S = 3 (C = 4) alone
    case("single_s3", modality(100, 100, 4, 1, n_out=100), B=3),
]

# geometries only the C ABI reaches: crops that are not centred, and resizes no reference expression gives
ABI_CASES = [
    # upsampling 100 -> 150 with the crop at the bottom-left corner: crop_y = rh - 64
    case("abi_bottom_left", modality(100, 100, 3, 1, geom=(150, 150, 86, 0)), modality(100, 100, 1, 0, geom=(150, 150, 0, 86))),
    # W = 3 stretched to 65536, the crop at its right edge: crop_x = rw - 64
    case("abi_w3_65536", modality(5, 3, 2, 1, geom=(64, 65536, 0, 65472)), modality(3, 5, 5, 0, geom=(65536, 64, 65472, 0))),
    # anisotropic 16 x 15.625 downsampling, and 1023 rows resized to 65536 with the crop at row 0 and a far column
    case("abi_aniso", modality(1024, 1000, 4, 1, geom=(64, 64, 0, 0)), modality(1023, 7, 8, 0, geom=(65536, 100, 0, 36))),
    # 480 x 640 at its reference resize, crop against the left and then the right edge
    case("abi_left_right", modality(480, 640, 3, 1, geom=(64, 85, 0, 0)), modality(480, 640, 1, 0, geom=(64, 85, 0, 21))),
]

# unread pixels set to NaN / +Inf: landscape, portrait and both 65536-long resizes
UNREAD_SHAPES = [(64, 1024), (1024, 64), (480, 640), (640, 480), (341, 256), (1, 1024), (1024, 1)]
# NaN in a pixel two overlapping upsampling bins read: 33 x 33 (bins of 1 and 2 rows and columns)
SHARED_PIXEL_SHAPE = (33, 33)

# batch identity: mixed geometry and channels, each input its own K split
IDENTITY_CASE = case("identity", modality(130, 70, 5, 1, n_out=100), modality(17, 900, 2, 0), B=160)
IDENTITY_BATCHES = (1, 3, 129)
# the largest batch: RGB-D at 96 x 128
MAX_B_CASE = case("max_b", modality(96, 128, 3, 1), modality(96, 128, 1, 0), B=1024)


def fused_cases():
    return SHAPE_CASES + PAIR_CASES + ABI_CASES
