"""Generates tests/golden/ref_pin_motions_320x240.npz: the reference-compiled side (oracle/_ref/liblsd_ref.so) of every comparison
of tests/test_ref_pin_motions.py, i.e. the case functions of tests/pin_cases.py and two constructed cases under the camera
motions of tests/motions.py, on the seeded 320x240 synthetic streams.  Written with save_npz_reproducible, so that a re-run
reproduces it byte for byte.
Run:  python -m tests.golden.make_golden_ref_pin_motions
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_pin_motions_320x240.npz")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from oracle import pyoracle
    from tests.golden.make_golden_ref_pin_globals import save_npz_reproducible
    pyoracle.build()
    if not pyoracle.ref_available():
        raise SystemExit("oracle/_ref is not built and the reference sources are absent: this fixture cannot be regenerated here")
    from tests import pin_cases
    res = pin_cases.record_motions()
    save_npz_reproducible(OUT, res)
    print(f"{OUT}: {len(res)} arrays")
