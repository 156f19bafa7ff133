"""Which regimes the train convs' plans reach, and that the layer-checked GPU cases reach every one of them.

tests/train_plan.py restates the host code that plans the train convs (choose_tile, the weight-gradient K split,
stat_blocks); test_gpu_train_shapes.py holds it to the library's own plan on the GPU.  Here, on the CPU, every
B <= 256 and T <= 1600 (a multiple of 16) is enumerated on the 132-SM H100 plan, and the case lists of
test_gpu_train_shapes.py must reach every regime found, each case at least one that no other case of its list reaches:
removing a case, or a change of the planning code that opens a new regime, turns this test red.
"""
import functools
from itertools import product

import pytest

from tests import test_gpu_backward_layer_parity as BWD
from tests import test_gpu_layer_parity as FWD
from tests import test_gpu_train_shapes as S
from tests import train_plan as P


@functools.lru_cache(maxsize=None)
def reachable(sync):
    return P.reachable(sync)


def cover(shapes, sync=False):
    return {c: P.case_regimes(*c, sync=sync) for c in shapes}


def assert_minimal(name, regs, within=None):
    """Every case of a list reaches a regime (of `within`, if given) that no other case of the list reaches."""
    for c, r in regs.items():
        others = set().union(*(v for d, v in regs.items() if d != c))
        own = (r - others) if within is None else (r & within) - others
        assert own, f"{name}: case {c} reaches nothing the other cases do not: removing it loses no regime"


def test_choose_tile_pads_least():
    """The restated box holds 128 pixels, spans the width, and pads the (h, n) grid least over every power-of-two
    split of the rows, ties to the taller box."""
    for B, H, W in product((1, 2, 3, 5, 9, 17, 33, 64, 128, 256), (1, 5, 17, 25, 31, 32, 50, 200, 800), (4, 8, 16, 32)):
        wt, hb, nb = P.choose_tile(B, H, W)
        assert wt == W and wt * hb * nb == 128
        rows = 128 // W
        pad = lambda h, n: -(-H // h) * h * (-(-B // n) * n)
        splits = [(1 << k, rows >> k) for k in range(rows.bit_length() - 1, -1, -1)]   # tallest first
        best = min(pad(h, n) for h, n in splits)
        assert (hb, nb) == next((h, n) for h, n in splits if pad(h, n) == best), (B, H, W)


def test_weight_gradient_slices_cover_every_chunk_once():
    for B, T in product((1, 3, 9, 17, 64, 256), (16, 80, 272, 400, 800, 1600)):
        for i in range(1, 12):
            p = P.layer_plan(i, B, T)
            ks, per, chunks = p["ksplit"], p["per"], p["chunks"]
            got = [min((k + 1) * per, chunks) - min(k * per, chunks) for k in range(ks)]
            assert sum(got) == chunks and max(got) == per, (B, T, i, got)
            assert 1 <= ks <= max(chunks // 4, 1)


def test_thirteen_box_shapes_are_reachable():
    shapes = sorted(r for r in reachable(False) if r[1].startswith("tile"))
    assert len(shapes) == 13, shapes


def test_fp16_cases_reach_every_regime_and_each_is_needed():
    regs = cover(S.FP16_SHAPES)
    missed = set(reachable(False)) - set().union(*regs.values())
    assert not missed, "unreached: " + "; ".join(f"stage {s} {r} (first at B, T = {reachable(False)[(s, r)]})"
                                                 for s, r in sorted(missed))
    assert_minimal("fp16", regs)


def test_bf16_cases_reach_every_box_the_earlier_checker_cases_never_built():
    earlier = set(FWD.TRAIN_CASES) | set(BWD.CASES)
    built = set().union(*(P.case_regimes(B, T) for _, B, T in earlier))
    never = {r for r in reachable(False) if r[1].startswith("tile")} - built
    assert never, "the earlier cases build every box shape: nothing for the bf16 cases to add"
    regs = cover(S.BF16_SHAPES)
    missed = never - set().union(*regs.values())
    assert not missed, f"bf16: boxes never layer-checked: {sorted(missed)}"
    assert_minimal("bf16", regs, within=never)


def test_synchronised_cases_reach_every_synchronised_regime():
    sync_only = {r for r in reachable(True) if "sync" in r[1]}
    assert sync_only, "no synchronised chain is longer than 64 terms"
    regs = cover(S.SYNC_SHAPES, sync=True)
    missed = sync_only - set().union(*regs.values())
    assert not missed, f"synchronised: unreached {sorted(missed)}"
    assert_minimal("synchronised", regs, within=sync_only)
