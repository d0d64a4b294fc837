"""Generate tests/golden/maps/* with the UNMODIFIED reference's map writers (datasets/data_io.py save_pfm / save_bin) and
record what its readers return (read_pfm / read_bin) in tests/golden/maps/expected.npz.

Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet):
    python tests/golden/make_mapio_golden.py <path to the reference checkout>"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "maps")
if len(sys.argv) != 2:
    raise SystemExit(__doc__)
sys.path.insert(0, os.path.abspath(sys.argv[1]))
from datasets import data_io as ref  # noqa: E402

os.makedirs(OUT, exist_ok=True)
rng = np.random.default_rng(20260923)
arrays = {
    "depth_hw": rng.uniform(425.0, 935.0, size=(23, 37)).astype(np.float32),
    "conf_hw1": rng.uniform(0.0, 1.0, size=(16, 20, 1)).astype(np.float32),
    "color_hw3": rng.normal(size=(9, 14, 3)).astype(np.float32),
}
arrays["depth_hw"][0, :4] = [0.0, -0.0, np.inf, np.nan]  # payload bytes must survive untouched
expected = {}
for name, arr in arrays.items():
    for ext in ("pfm", "bin"):
        path = os.path.join(OUT, f"{name}.{ext}")
        ref.save_map(path, arr)
        back = ref.read_map(path)
        expected[f"{name}.{ext}"] = back
        assert back.dtype == np.float32 and back.ndim == 3
    expected[f"{name}.input"] = arr
# a big-endian PFM with a non-unit scale, the way a foreign writer produces it (header by hand, payload via numpy)
be = rng.uniform(0, 10, size=(5, 7)).astype(np.float32)
with open(os.path.join(OUT, "foreign_be.pfm"), "wb") as f:
    f.write(b"Pf\n7 5\n2.5\n")
    np.flipud(be).astype(">f4").tofile(f)
got, scale = ref.read_pfm(os.path.join(OUT, "foreign_be.pfm"))
assert scale == 2.5 and np.array_equal(got[..., 0], be)
expected["foreign_be.pfm"] = np.ascontiguousarray(got).astype(np.float32)
np.savez_compressed(os.path.join(OUT, "expected.npz"), **expected)
print("wrote", sorted(os.listdir(OUT)))
