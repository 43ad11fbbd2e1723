"""Cases of tests/test_gpu_scale_space.py and the launch geometry of `blur_kernel` (pyramid.cu), shared with the CPU test that asserts
which input fill and output store paths those cases reach.  Sizes are in floats; a torch allocation starts 16-byte aligned."""
import collections

# ---- ag_gaussian_blur ----------------------------------------------------------------------------------------------------------
RADII = list(range(1, 13))
BLUR_SHAPES = [(1, 1), (1, 9), (9, 1), (3, 5),          # smaller than the radius
               (63, 64), (64, 64), (65, 67),            # around the 64 x 64 tile
               (37, 41), (37, 42), (37, 43),            # w % 4 = 1, 2, 3
               (200, 328)]                              # interior tiles in both directions at R = 12
BLUR_BATCHES = (1, 3)
# (h, w) x (input offset, output offset) in floats into a larger allocation, at radii OFFSET_RADII
OFFSET_SHAPES = [(64, 64), (65, 68), (37, 43), (200, 328)]
OFFSETS = [(k, 0) for k in (1, 2, 3)] + [(0, k) for k in (1, 2, 3)] + [(k, k) for k in (1, 2, 3)]
OFFSET_RADII = (1, 4, 12)


def sigma_for_radius(R):
    """k = int(6 sigma + 1) = 2R + 1 taps."""
    return (R + 0.25) / 3.0


# ---- ag_pyramid_build ----------------------------------------------------------------------------------------------------------
GRAF = (256, 320)   # tests/golden/graf_crop.npz
# (name, B, H, W, nlevels, init_sigma, border); name "graf" takes the graf crop (B = 1), the others seeded noise
PYR_CASES = ([("noise", 1, 97, 127, nl, s, 5) for nl in (2, 3, 4, 5, 6) for s in (0.5, 1.0, 1.6, 2.0)]
             + [("noise", 1, 97, 127, 1, 1.0, 5), ("noise", 1, 97, 127, 1, 1.6, 5), ("noise", 1, 97, 127, 1, 2.0, 5)]
             + [("graf", 1) + GRAF + (3, 1.6, b) for b in (0, 5, 33)]
             + [("graf", 1) + GRAF + (5, 1.0, 5)]
             + [("noise", 2, 97, 127, 3, 1.6, 5), ("noise", 2, 97, 127, 2, 2.0, 0), ("noise", 2, 97, 127, 6, 0.5, 33),
                ("noise", 2, 97, 127, 4, 1.0, 5)]
             + [("noise", 1, 767, 1023, 3, 1.6, 5), ("noise", 1, 767, 1023, 5, 1.0, 0)])
NO_TMA_PYR_CASES = [("graf", 1) + GRAF + (3, 1.6, 5), ("noise", 2, 97, 127, 3, 1.6, 5), ("noise", 1, 767, 1023, 3, 1.6, 5)]
NO_TMA_BLUR_CASES = [(3, 200, 328, R) for R in (1, 6, 12)]                                # AG_BLUR_NO_TMA=1 subprocess
BATCH_CASE = (3, 97, 127, 3, 1.6, 5)                                                       # == three B = 1 pyramids

MAX_TAPS = 25


def pyramid_blurs(plan):
    """The blur_kernel launches of ag_pyramid_build: (h, w, sigma, input offset, output offset), offsets in floats
    from the pyramid buffer (None: the input image)."""
    out = []
    for o in range(plan.n_octaves):
        h, w = plan.h[o], plan.w[o]
        if o == 0 and plan.blur_sigma[0][0] > 0.0:
            out.append((h, w, plan.blur_sigma[0][0], None, plan.level_offset[0][0]))
        for l in range(1, plan.n_levels):
            out.append((h, w, plan.blur_sigma[o][l], plan.level_offset[o][l - 1], plan.level_offset[o][l]))
    return out


# ---- blur_kernel's per-tile paths ------------------------------------------------------------------------------------------------
TW = TH = 64


def blur_tile_paths(B, h, w, R, in_off=0, out_off=0, tma=True):
    """Counter of the input fill ("tma", "bulk", "ldg128", "scalar") and output store ("store_v4", "store_scalar") of every CTA of one
    blur_kernel<R> launch whose input / output start at in_off / out_off floats from a 16-byte boundary (pyramid.cu, step 1 and 3)."""
    R4 = (R + 3) // 4 * 4
    IW = ((TW + 2 * R + 3) // 4 + 1) * 4
    IH = TH + 2 * R
    c = collections.Counter()
    nx, ny = -(-w // TW), -(-h // TH)
    for b in range(B):
        img_aligned = (in_off + b * h * w) % 4 == 0
        for by in range(ny):
            for bx in range(nx):
                x0, y0 = bx * TW, by * TH
                wide = w % 4 == 0 and x0 - R4 >= 0 and x0 - R4 + IW <= w and img_aligned
                bulk = wide and y0 - R >= 0 and y0 - R + IH <= h
                tmap = tma and w % 4 == 0 and in_off % 4 == 0 and IW <= 256 and IH <= 256
                c["tma" if bulk and tmap else "bulk" if bulk else "ldg128" if wide else "scalar"] += 1
                c["store_v4" if w % 4 == 0 and out_off % 4 == 0 else "store_scalar"] += 1
    return c


def misaligned_levels(plan):
    """(octave, level) of the levels blur_kernel writes whose width is a multiple of 4 but whose start is not 16-byte aligned."""
    return [(o, l) for o in range(plan.n_octaves) for l in range(plan.n_levels)
            if plan.w[o] % 4 == 0 and plan.level_offset[o][l] % 4 != 0 and (l > 0 or (o == 0 and plan.blur_sigma[0][0] > 0.0))]
