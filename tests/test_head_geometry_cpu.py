"""The head's host-side geometry constants (odise_b200/head.py::pos_sine, ::ref_points) against the oracle's
(oracle/m2f.py, pinned to the reference's PositionEmbeddingSine / get_reference_points by tests/test_oracle_cpu.py) at
portrait, landscape, odd and square maps: both normalise rows by H and columns by W, so a swap shows only at H != W."""
import pytest
import torch

from odise_b200 import head
from oracle import m2f

SHAPES = [(18, 14), (14, 18), (7, 9), (16, 16)]


@pytest.mark.parametrize("hw", SHAPES)
def test_pos_sine_matches_oracle(hw):
    H, W = hw
    got = head.pos_sine(H, W)                                               # token-major [H*W, 256]
    want = m2f.position_embedding_sine(1, H, W)[0].flatten(1).t()           # NCHW [1, 256, H, W] -> [H*W, 256]
    assert got.shape == (H * W, 256)
    assert (got - want).abs().max().item() <= 1e-6                          # same fp32 recipe: 1e-6 absolute


def test_ref_points_matches_oracle():
    for shapes in ([(18, 14), (36, 28), (72, 56)], [(14, 18), (7, 9), (16, 16)]):
        got = head.ref_points(shapes)                                       # [S, L, 2]
        want = m2f.reference_points(shapes, 1)[0]                           # [1, S, L, 2]
        assert got.shape == want.shape == (sum(h * w for h, w in shapes), len(shapes), 2)
        assert (got - want).abs().max().item() <= 1e-6                      # (x / W, y / H) per level: 1e-6 absolute
