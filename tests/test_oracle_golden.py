"""Pin the CPU oracle to the reference's OWN golden images (SURVEY.md 8c).

Each test renders one scene of tests/reference_goldens.py with the oracle and compares the Rgba8UnormSrgb result
with the decoded reference PNG by that scene's criterion.
"""
import pytest

import reference_goldens as scenes
from rend3_b200.world import LEFT, RIGHT

from oracle import load_oracle_backend


def test_empty():
    scenes.empty(load_oracle_backend)


@pytest.mark.parametrize(
    "handedness,winding,visible",
    [(LEFT, "Cw", True), (LEFT, "Ccw", False), (RIGHT, "Cw", False), (RIGHT, "Ccw", True)],
)
def test_triangle(handedness, winding, visible):
    scenes.triangle(load_oracle_backend, handedness, winding, visible)


def test_coordinate_space():
    scenes.coordinate_space(load_oracle_backend)


@pytest.mark.parametrize("samples", [1, 4])
def test_sample_coverage(samples):
    scenes.sample_coverage(load_oracle_backend, samples)


def test_msaa_four():
    scenes.msaa_four(load_oracle_backend)


def test_multi_frame_add():
    scenes.multi_frame_add(load_oracle_backend)


def test_duplicate_object_retain():
    scenes.duplicate_object_retain(load_oracle_backend)


def test_shadow_plane():
    scenes.shadow_plane(load_oracle_backend)


def test_shadow_cube():
    scenes.shadow_cube(load_oracle_backend)


def test_cube_example_screenshot():
    scenes.cube_example_screenshot(load_oracle_backend)
