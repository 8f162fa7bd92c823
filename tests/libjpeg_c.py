"""libjpeg-turbo's C decode path, as a reference for files whose IDCT leaves the +-512 range.

``decode_c(files)`` decodes JPEG byte strings as ``np.asarray(PIL.Image.open(...).convert("RGB"))`` does, in a child
Python process started with ``JSIMD_FORCENONE=1``.  With that variable libjpeg-turbo runs no SIMD code: the IDCT is
``jidctint.c`` (each output wrapped to 10 bits, ``idct_range_limit[x & 1023]``), upsampling ``jdsample.c`` and colour
conversion ``jdcolor.c``, the functions ``defer_b200.jpeg`` follows beyond the range.  The SIMD IDCT that Pillow runs
on x86 by default saturates instead of wrapping, so it gives other pixels there.

libjpeg-turbo reads the variable once per process, and this process may already have decoded with SIMD; hence the child.
It gets the files and returns the images through ``.npz`` files in a temporary directory, and exits before ``decode_c``
returns.

``decode_c`` skips the calling test when Pillow is missing or is not built against libjpeg-turbo 3.1, and fails it when
the child does not take the C path: a one-block file whose DC-only IDCT output is 128 + 1100 must decode to 204, as
``idct_range_limit[1100 & 1023]`` gives (the SIMD IDCT gives 0).
"""
from __future__ import annotations

import os
import subprocess
import sys
import tempfile
from pathlib import Path
from typing import List, Sequence

import numpy as np
import pytest

import jpeg_craft as jc

_CHILD = r"""
import io, sys
import numpy as np
from PIL import Image, features
src = np.load(sys.argv[1])
out = {k: np.asarray(Image.open(io.BytesIO(src[k].tobytes())).convert("RGB")) for k in src.files}
np.savez(sys.argv[2], version=np.array(features.version_feature("libjpeg_turbo")), **out)
"""

#: the sentinel's DC coefficient and quantiser: x = 110 * 80 / 8 = 1100, idct_range_limit[1100 & 1023] = 204
SENTINEL_DC, SENTINEL_Q, SENTINEL_PIXEL = 110, 80, 204


def _check_pillow() -> str:
    pytest.importorskip("PIL.Image")
    from PIL import features
    if not features.check_feature("libjpeg_turbo"):
        pytest.skip("Pillow is not built against libjpeg-turbo")
    version = features.version_feature("libjpeg_turbo") or ""
    if not version.startswith("3.1."):
        pytest.skip(f"Pillow bundles libjpeg-turbo {version}, not 3.1.x")
    return version


def sentinel() -> bytes:
    """An 8x8 grayscale file of one DC-only block whose IDCT output is 128 + 1100 everywhere."""
    coef = np.zeros((1, 64), np.int32)
    coef[0, 0] = SENTINEL_DC
    return jc.craft(8, 8, "gray", [np.full(64, SENTINEL_Q)], [jc.one_symbol(7)], [jc.one_symbol(0)], coef=coef)


def _run(files: Sequence[bytes]) -> tuple:
    with tempfile.TemporaryDirectory() as tmp:
        src, dst = Path(tmp) / "in.npz", Path(tmp) / "out.npz"
        np.savez(src, **{f"f{i}": np.frombuffer(bytes(d), np.uint8) for i, d in enumerate(files)})
        env = dict(os.environ, JSIMD_FORCENONE="1")
        flags = ["-s"] if sys.flags.no_user_site else []         # the same Pillow as this process
        r = subprocess.run([sys.executable, *flags, "-c", _CHILD, str(src), str(dst)], env=env, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        with np.load(dst) as z:
            return str(z["version"]), [z[f"f{i}"] for i in range(len(files))]


def decode_c(files: Sequence[bytes]) -> List[np.ndarray]:
    """uint8 RGB ``(h, w, 3)`` of each file as libjpeg-turbo's C path decodes it through Pillow."""
    version = _check_pillow()
    child, out = _run([sentinel()] + list(files))
    assert child == version, (child, version)
    got = np.unique(out[0])
    assert got.tolist() == [SENTINEL_PIXEL], (
        f"JSIMD_FORCENONE=1 did not select libjpeg-turbo's C IDCT: the sentinel decodes to {got.tolist()}, "
        f"not {SENTINEL_PIXEL}")
    return out[1:]
