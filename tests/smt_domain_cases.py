"""The accuracy cases of tests/test_gpu_smt_domain.py as plain data, shared with tests/test_smt_host.py, which checks
through a restatement of the host's tiling that they reach every kernel's tile edges.

A case is a dict: the stand-in's shape (``D``, ``pose_index`` or None, ``d_model``, ``nhead``, ``pretraining``), the
batch (``B``, ``M``) and ``valid``, the number of valid memory slots of each env (its token count is one more: the
current token is always valid; under pretraining it is the only one).
"""

# (d_model, nhead): head dims 1, 8, 9, 32, 25, 64, 128, 125 and 8; d below 32, d not a multiple of 32, and d, 2d and
# 3d ending in a partial 128-column tile (d = 384 and 512 end in a full one)
WIDTHS = ((8, 8), (24, 3), (72, 8), (96, 3), (200, 8), (320, 5), (384, 3), (500, 4), (512, 64))
# fusion_encoder[0] widths around the 64-wide K tiles: without pose encoding F = D ...
NO_POSE_D = (1, 2, 63, 64, 65, 1023, 1024)
# ... and with it F = pose_index + 16 (16, 63, 64, 65, 77 and 1036, the fuse kernel's largest X tile)
POSE_INDICES = (0, 47, 48, 49, 61, 1020)
# (pose_index, D) with D > pose_index + 4: NaN in the columns past the pose must not reach the output
TRAILING = ((0, 9), (48, 100))
# per-env token counts (current token included) at the 16-row query tiles and 64-key key tiles, in one batch
COUNTS = (1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1023, 1024)
LAYOUTS = ("contiguous", "wrapped", "scattered")
DECODER_B = (1, 2, 3, 5, 1023)
# one env placed at positions 0..3 of the second 4-env decoder group and across the last, partial group of 11
PROBE_B = 11
PROBE_POSITIONS = (4, 5, 6, 7, 8, 9, 10)
MASK_VALUES = (1.0, 2.0, 0.5, 0.0, -1.0, float("inf"), float("-inf"), float("nan"))
# eps of enc norm1, norm2, encoder.norm, dec norm1, norm2, norm3, decoder.norm
EPS = (1e-4, 1e-8, 1e-3, 1e-5, 1e-6, 1e-7, 3e-4)
SCALES = (1e-6, 1e3)
LARGEST_B = 1024


def default_valid(B, M):
    """make_inputs' default: env n holds M (n + 1) / (B + 1) valid slots."""
    return [(M * (n + 1)) // (B + 1) for n in range(B)]


def case(name, B, M, D=70, pose_index=60, d_model=64, nhead=4, valid=None, pretraining=False, **extra):
    c = dict(name=name, B=B, M=M, D=D, pose_index=pose_index, d_model=d_model, nhead=nhead, pretraining=pretraining,
             valid=list(default_valid(B, M) if valid is None else valid))
    c.update(extra)
    return c


def width_cases():
    return [case(f"d{d}h{h}", 5, 40, d_model=d, nhead=h, seed=d + h) for d, h in WIDTHS]


def fusion_cases():
    out = [case(f"D{D}", 5, 20, D=D, pose_index=None, seed=D) for D in NO_POSE_D]
    out += [case(f"pi{p}", 5, 20, D=p + 4, pose_index=p, seed=p) for p in POSE_INDICES]
    out += [case(f"pi{p}D{D}", 5, 20, D=D, pose_index=p, seed=p + D) for p, D in TRAILING]
    return out


def count_cases():
    """All 16 counts in one batch of M = 1023 slots (hd 32), in each slot layout."""
    return [case(f"counts_{lay}", len(COUNTS), 1023, D=40, pose_index=36, d_model=96, nhead=3,
                 valid=[c - 1 for c in COUNTS], layout=lay, seed=60 + i) for i, lay in enumerate(LAYOUTS)]


def largest_cases():
    """The largest attention / decoder tiles (d 512, hd 128, every one of 1023 slots valid: 16 key tiles), the largest
    fuse tile (D 1024, pose index 1020, d 512), and the most envs with the most tokens at a small d."""
    return [case("attn_1024", 2, 1023, d_model=512, nhead=4, valid=[1023, 1023], seed=70),
            case("fuse_1036", 3, 40, D=1024, pose_index=1020, d_model=512, nhead=4, seed=71),
            case("envs_1024", LARGEST_B, 1023, D=12, pose_index=8, d_model=32, nhead=4,
                 valid=[(389 * b) % 1024 for b in range(LARGEST_B)], seed=72)]


def decoder_cases():
    return [case(f"B{B}", B, 10, D=20, pose_index=16, d_model=40, nhead=5, seed=80 + B) for B in DECODER_B]


def probe_cases():
    return [case(f"probe{p}", PROBE_B, 30, D=20, pose_index=16, d_model=40, nhead=5, seed=90, probe=p)
            for p in PROBE_POSITIONS]


def mask_cases():
    """Every mask value in every env (valid slots counted by the stand-in's rule: padding iff 1 - m > 0), and
    pretraining with a goal and non-zero masks (only the current token)."""
    B, M = 6, 48
    n_valid = sum(1 for v in MASK_VALUES if not (1.0 - v > 0))           # 1, 2, +inf and NaN
    return [case("mask_values", B, M, valid=[M // len(MASK_VALUES) * n_valid] * B, seed=100),
            case("pretraining", B, M, pretraining=True, valid=[0] * B, seed=101)]


def numeric_cases():
    out = [case("eps", 6, 40, d_model=72, nhead=8, seed=110),
           case("constant_norm1", 6, 40, d_model=72, nhead=8, seed=111)]
    out += [case(f"scale{s:g}", 6, 40, d_model=72, nhead=8, seed=112, scale=s) for s in SCALES]
    out.append(case("pose_edges", 8, 12, d_model=72, nhead=8, valid=[12] * 8, seed=114))
    return out


def sweep():
    """Every accuracy case the GPU file runs."""
    return (width_cases() + fusion_cases() + count_cases() + largest_cases() + decoder_cases() + probe_cases()
            + mask_cases() + numeric_cases())
