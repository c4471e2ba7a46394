#!/usr/bin/env python
"""Vendor the UNMODIFIED reference package into the git-ignored oracle/_ref (called by build()).

    python oracle/vendor_ref.py [--force]     # <reference>/bayes_opt -> oracle/_ref/bayes_opt

The drop-in tests, the reference arm of bench.py and the reference's own test modules need the
reference package `bayes_opt` importable; it is not a dependency of the product and is not on PyPI
in this environment, so it is copied byte for byte from a reference checkout (B200BO_REFERENCE)
into oracle/_ref, which is never part of the history.  Nothing is edited.  Two things the reference
needs at import time are supplied beside it (they are not reference code):

  * `colorama` (imported by bayes_opt/target_space.py and logger.py) -> the stub from oracle/shims/colorama
  * package metadata: bayes_opt/__init__.py asks importlib.metadata for the version of the
    distribution "bayesian-optimization" -> a minimal `*.dist-info/METADATA` with the version of the
    reference's pyproject.toml, so that putting oracle/_ref on sys.path is all a caller does.

Product code (bayesianoptimization_b200/) never reads oracle/_ref: it imports `bayes_opt` from wherever
the user's environment provides it; tests/conftest.py and bench.py put oracle/_ref on sys.path.
"""
from __future__ import annotations

import os
import re
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("B200BO_REFERENCE", "/root/reference")
DST = os.path.join(ROOT, "oracle", "_ref")
# the reference's test modules that exercise the hot path and its callers (SURVEY.md 8a/8c)
REF_TESTS = ("test_acquisition.py", "test_constraint.py", "test_bayesian_optimization.py", "test_target_space.py",
             "test_seq_domain_red.py", "test_parameter.py", "test_util.py", "test_logger.py")


def reference_version() -> str:
    txt = open(os.path.join(REF, "pyproject.toml")).read()
    m = re.search(r'^version\s*=\s*"([^"]+)"', txt, re.M)
    return m.group(1) if m else "0"


def _make_writable(path: str) -> None:
    for base, dirs, files in os.walk(path):
        for n in dirs + files:
            q = os.path.join(base, n)
            os.chmod(q, os.stat(q).st_mode | 0o200)
    os.chmod(path, os.stat(path).st_mode | 0o200)


def vendor(force: bool = False) -> str | None:
    """Returns the vendored path, or None when neither the reference checkout nor an earlier copy is present."""
    src = os.path.join(REF, "bayes_opt")
    if not os.path.isdir(src):
        return DST if os.path.isdir(os.path.join(DST, "bayes_opt")) else None
    stamp = os.path.join(DST, ".vendored")
    ver = reference_version()
    if (not force and os.path.exists(stamp) and open(stamp).read().strip() == ver
            and all(os.path.exists(os.path.join(DST, "ref_tests", t)) for t in REF_TESTS)):
        return DST
    if os.path.isdir(DST):
        _make_writable(DST)
        shutil.rmtree(DST)
    os.makedirs(DST)
    shutil.copytree(src, os.path.join(DST, "bayes_opt"), ignore=shutil.ignore_patterns("__pycache__"))
    shutil.copytree(os.path.join(ROOT, "oracle", "shims", "colorama"), os.path.join(DST, "colorama"),
                    ignore=shutil.ignore_patterns("__pycache__"))
    _make_writable(DST)  # the reference checkout may be read-only and copytree keeps the modes
    # the reference's own tests for the path: run against the drop-in (tests/test_gpu_reference_suite.py)
    tdst = os.path.join(DST, "ref_tests")
    os.makedirs(tdst)
    for name in REF_TESTS:
        shutil.copy(os.path.join(REF, "tests", name), os.path.join(tdst, name))
    _make_writable(DST)
    info = os.path.join(DST, f"bayesian_optimization-{ver}.dist-info")
    os.makedirs(info)
    with open(os.path.join(info, "METADATA"), "w") as f:
        f.write(f"Metadata-Version: 2.1\nName: bayesian-optimization\nVersion: {ver}\n")
    with open(os.path.join(info, "RECORD"), "w") as f:
        f.write("")
    with open(stamp, "w") as f:
        f.write(ver + "\n")
    return DST


if __name__ == "__main__":
    p = vendor(force="--force" in sys.argv)
    print(p if p else "reference tree not present; nothing vendored")
