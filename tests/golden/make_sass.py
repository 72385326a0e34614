#!/usr/bin/env python3
"""Generates tests/golden/sass.json — the count and sha256 of every function's SASS in the built libcdprobe.so, which
tests/test_sass_pins_cpu.py holds the library to.  A change that alters a kernel on purpose reruns this after building
(CUDA 12.9), and the diff of sass.json names exactly the functions that moved.

Run:  python tests/golden/make_sass.py   (after the library is built; rewrites sass.json deterministically)
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

import cdprobe_pkg  # noqa: E402
from kernel_tools import sass_pins  # noqa: E402


def main():
    lib = cdprobe_pkg.load().abi.LIB_PATH
    path = os.path.join(HERE, "sass.json")
    with open(path, "w") as f:
        json.dump(sass_pins(lib), f, indent=1, sort_keys=True)
        f.write("\n")
    print(path)


if __name__ == "__main__":
    main()
