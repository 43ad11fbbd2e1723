"""CPU tests for the inputs tests/test_gpu_detect.py feeds the detector: the adversarial pyramids must reach every branch of the level-drop
rule (a level with <= 1 positive maximum is dropped, HandCraftedModules.py:253), and the selection rule the GPU output is held to must be
what the oracle's multi_scale_detector returns.  Without the first, the GPU test could silently drift into testing only the branch where
every level is accepted."""
import collections
import itertools

import affnet_oracle as O
from helpers import ADV_H, ADV_W, OracleCandidates, adversarial_pyramid, detector_level_stats

ADV_SEEDS = range(400)
MR = 5.192


def _sigmas(nlevels):
    sizes, _, sig, _ = O.pyramid_plan(ADV_H, ADV_W, nlevels, 1.6, 5)
    assert sizes == [(40, 40), (20, 20)]
    return sig


def test_adversarial_pyramids_cover_the_level_drop_rule():
    sig = _sigmas(3)
    combos, n_pos, negs, wraps = collections.Counter(), collections.Counter(), 0, 0
    for seed in ADV_SEEDS:
        pyr = adversarial_pyramid(seed)
        st = detector_level_stats(pyr[0], sig[0], MR)
        combos[tuple(int(s[1]) for s in st)] += 1
        for p, acc, neg, wrap in st:
            n_pos[min(p, 3)] += 1
            negs += neg
            wraps += wrap
            assert acc == (p > 1)
    print("\noctave 0 (a1, a2, a3) accept combinations:", sorted(combos.items()), " levels by n_pos (3 = >= 3):", sorted(n_pos.items()),
          " levels with negative masked responses:", negs, " accepted levels whose map wrapped:", wraps)
    assert set(combos) == set(itertools.product((0, 1), repeat=3))
    assert combos[(0, 0, 0)] >= 10
    assert n_pos[0] >= 10 and n_pos[1] >= 10 and n_pos[2] >= 10
    assert negs >= 10 and wraps >= 10


def test_adversarial_pyramids_at_other_level_counts_drop_levels():
    for nlevels in (1, 2, 4, 5, 6):
        sig = _sigmas(nlevels)
        acc = collections.Counter()
        for seed in ADV_SEEDS[:100]:
            pyr = adversarial_pyramid(seed, nlevels)
            assert len(pyr[0]) == nlevels + 2
            for p, a, _, _ in detector_level_stats(pyr[0], sig[0], MR):
                acc[a] += 1
        assert acc[True] >= 20 and acc[False] >= 20, (nlevels, acc)


def test_selection_rule_is_the_oracles():
    """OracleCandidates.select(nf) (top nf by response, then seq; or all in seq order) against multi_scale_detector(nf) at the edges of
    the sorted / unsorted switch, on pyramids that drop levels, trim levels and drop everything."""
    sig = _sigmas(3)
    seen = collections.Counter()
    for seed in ADV_SEEDS[:120]:
        c = OracleCandidates(adversarial_pyramid(seed), sig, MR)
        T = c.total
        seen["empty" if T == 0 else "some"] += 1
        for nf in sorted({1, 2, T - 1, T, T + 1, 0, -1}):
            c.check_against_oracle(nf)
            seen["sorted" if c.order(nf)[1] else "unsorted"] += 1
    assert seen["empty"] > 0 and seen["sorted"] > 0 and seen["unsorted"] > 0, seen
