"""Generates tests/golden/ref_pin_globals_320x240.npz: the reference-compiled side (oracle/_ref/liblsd_ref.so) of every comparison
of tests/test_ref_pin_globals.py, i.e. the case functions of tests/pin_cases.py under non-default run-time settings, on the
seeded 320x240 synthetic stream.  The archive is written with fixed member timestamps and in key order, so that a re-run
reproduces it byte for byte.
Run:  python -m tests.golden.make_golden_ref_pin_globals
"""
import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_pin_globals_320x240.npz")


def save_npz_reproducible(path, arrays):
    """np.savez_compressed's layout (one .npy member per key) without its wall-clock member timestamps"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            z.writestr(info, buf.getvalue())


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from lsd_slam_b200 import synth
    from oracle import pyoracle
    pyoracle.build()
    if not pyoracle.ref_available():
        raise SystemExit("oracle/_ref is not built and the reference sources are absent: this fixture cannot be regenerated here")
    from tests import pin_cases
    seq = synth.Sequence(320, 240, seed=1234)
    frames = {k: seq.render(k) for k in range(26)}
    res = pin_cases.record_globals(seq, frames)
    save_npz_reproducible(OUT, res)
    print(f"{OUT}: {len(res)} arrays")
