"""Every function in the built libcdprobe.so compiles to the SASS pinned in tests/golden/sass.json (count and sha256 of
its instructions as kernel_sass reads them, CUDA 12.9), and no function is added or removed unpinned.  A change that
alters a kernel on purpose regenerates the pins with tests/golden/make_sass.py, so the diff names the kernels that
moved."""
import json
import os

import pytest

from conftest import ROOT
from kernel_tools import sass_pins

GOLDEN = os.path.join(ROOT, "tests", "golden", "sass.json")


@pytest.fixture(scope="module")
def pins(pkg):
    return sass_pins(pkg.abi.LIB_PATH)


def test_the_library_holds_exactly_the_pinned_functions(pins):
    want = json.load(open(GOLDEN))
    assert sorted(pins) == sorted(want)


@pytest.mark.parametrize("name", sorted(json.load(open(GOLDEN))))
def test_each_function_compiles_to_its_pinned_sass(pins, name):
    assert pins.get(name) == json.load(open(GOLDEN))[name]
