"""Write tests/golden/phase_a_bits.npz: the bits of phase A's covariance results that tests/test_gpu_phase_a_bits.py
holds every later build to (what is recorded: that file's docstring).

  python tools/phase_a_bits.py [--root TREE] [--out tests/golden/phase_a_bits.npz] [--check]

--root imports bayesianoptimization_b200 (and its built library) from another checkout, e.g. the commit before a
change to the covariance arithmetic, so the fixture comes from the code the change must reproduce.  --check compares
against an existing file instead of writing it and prints the names that differ.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT, help="checkout whose bayesianoptimization_b200 computes the bits")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "phase_a_bits.npz"))
    ap.add_argument("--check", action="store_true", help="compare with --out instead of writing it")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    sys.path.insert(1, os.path.join(ROOT, "tests"))
    import bayesianoptimization_b200 as bo

    import test_gpu_phase_a_bits as T

    print(f"library: {bo._lib.LIB_PATH}", flush=True)
    z = T.pack(T.compute(bo))
    if args.check:
        with np.load(args.out, allow_pickle=False) as f:
            bad = [k for k in sorted(set(z) | set(f.files)) if k not in f.files or k not in z
                   or not np.array_equal(z[k], f[k])]
        print(f"{len(z)} arrays, {len(bad)} differ: {bad}")
        sys.exit(1 if bad else 0)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    np.savez(args.out, **z)
    print(f"wrote {args.out}: {len(z)} arrays, {os.path.getsize(args.out)} bytes")


if __name__ == "__main__":
    main()
