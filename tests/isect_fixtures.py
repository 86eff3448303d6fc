"""Inputs of the intersect stage that take the depth sort's rarely-used branches (numpy, seeded).

The depth order of the planned intersect path is a stable LSD radix sort of the float32 depth bits, 8 bits per pass,
that skips every pass whose digit is the same for all Gaussians with at least one tile (gsb_devsort.cuh,
radix_pass_skipped).  Random depths skip only pass 3, the exponent byte.  Each fixture here is named for the set of
passes it makes the sort skip; skip_pattern() restates the rule so a test can check that a fixture really does.
"""
from __future__ import annotations

import numpy as np

# gsb_intersect.cu kMaxWindowTiles: more (camera, tile) pairs than this and the histogram and placement run as several
# launches over windows of tiles
WINDOW_TILES = 36 * 1024


def skip_pattern(depths, active) -> tuple:
    """Passes (0 = low byte .. 3 = sign and exponent) that the depth sort skips: those whose 8-bit digit agrees over
    the depth bits of every active Gaussian (OR and AND of the keys agree on the byte).  No active Gaussian: none."""
    keys = np.ascontiguousarray(depths, np.float32).reshape(-1).view(np.uint32)[np.asarray(active).reshape(-1)]
    k_or = int(np.bitwise_or.reduce(keys)) if keys.size else 0
    k_and = int(np.bitwise_and.reduce(keys)) if keys.size else 0xFFFFFFFF
    return tuple(p for p in range(4) if ((k_or ^ k_and) >> (8 * p)) & 0xFF == 0)


def _bits(u32):
    return np.asarray(u32, np.uint32).view(np.float32)


def _f32_bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _one_depth(n, rng):
    return np.full(n, 2.75, np.float32)


def _integers(n, rng):  # integers 1..1000: the low byte of the mantissa is zero, every other byte varies
    return np.concatenate([np.float32([1.0, 257.0, 3.0]), rng.integers(1, 1001, n).astype(np.float32)])[:n]


def _sixty_fourths(n, rng):  # 2 + k/64, k < 128: only byte 2 (exponent LSB and the top mantissa bits) varies
    k = np.concatenate([[0, 1, 127], rng.integers(0, 128, n)])[:n]
    return (2.0 + k / 64.0).astype(np.float32)


def _middle_byte_fixed(n, rng):  # [1, 8) with byte 1 forced to 0x5a: bytes 0, 2 and 3 vary
    u = _f32_bits(rng.random(n, dtype=np.float32) * 7.0 + 1.0)
    u = np.concatenate([np.uint32([0x3F805A00, 0x40A15A37, 0x3FC05A11]), u])[:n]
    return _bits((u & np.uint32(0xFFFF00FF)) | np.uint32(0x5A00))


def _random_octave(n, rng):  # uniform in [2, 4): what a typical scene gives, only the exponent byte is constant
    w = _bits(np.uint32([0x40000000, 0x40123456, 0x40654321]))
    return np.concatenate([w, (rng.random(n, dtype=np.float32) * 2.0 + 2.0)]).astype(np.float32)[:n]


# fixture name -> (generator of the active Gaussians' depths, passes the sort skips on them)
DEPTHS = {
    "skip_all": (_one_depth, (0, 1, 2, 3)),
    "skip_0": (_integers, (0,)),
    "skip_013": (_sixty_fourths, (0, 1, 3)),
    "skip_1": (_middle_byte_fixed, (1,)),
    "skip_3": (_random_octave, (3,)),
}


def intersect_inputs(name, C, N, width, height, tile_size=16, seed=0, max_radius=40):
    """(means2d [C,N,2] f32, radii [C,N,2] i32, depths [C,N] f32, active [C,N] bool) for intersect_tile.

    Active Gaussians have on-screen means and radii in [1, max_radius] pixels; their depths, in flattened order, come
    from fixture `name`.  When N > 1, every third Gaussian is inactive, alternately with zero radii and with a box
    that clamps to zero tiles off the right or bottom edge.  The inactive ones get random depths that differ in every
    byte, so the sort must ignore them to skip what the fixture names."""
    gen, _ = DEPTHS[name]
    rng = np.random.default_rng(seed)
    n = C * N
    means2d = np.stack([rng.random(n) * width, rng.random(n) * height], -1).astype(np.float32)
    radii = rng.integers(1, max_radius + 1, (n, 2)).astype(np.int32)
    inactive = (np.arange(n) % 3 == 1) if N > 1 else np.zeros(n, bool)
    depths = np.empty(n, np.float32)
    depths[inactive] = (rng.random(int(inactive.sum())) * 50.0 + 0.3).astype(np.float32)
    depths[~inactive] = gen(int((~inactive).sum()), rng)
    zero_r = inactive & (np.arange(n) % 2 == 0)
    off = inactive & ~zero_r
    radii[zero_r] = 0
    # box entirely past the last tile column or row: x0 = x1 = tile_width (or the same for y), zero tiles
    far = rng.random(int(off.sum())) < 0.5
    m_off = means2d[off]
    m_off[far, 0] = width + tile_size + max_radius + rng.random(int(far.sum())) * 100
    m_off[~far, 1] = height + tile_size + max_radius + rng.random(int((~far).sum())) * 100
    means2d[off] = m_off
    active = ~inactive
    return (means2d.reshape(C, N, 2), radii.reshape(C, N, 2), depths.reshape(C, N), active.reshape(C, N))
