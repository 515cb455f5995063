"""Writes tests/golden/rawint4_pack.npz: the compressed-tensors INT4 format pinned by the package that defines it.

A few rows of known int8 values in -8..7 (every value in every word position) are packed by
compressed_tensors.pack_to_int32(num_bits=4) and stored next to the values and bf16 scale bits, so that the format tests
run where the package is not installed.  Re-running this script rewrites the file byte for byte (fixed seed, fixed zip
timestamps): a diff in the .npz means the package packs differently.

    python tests/golden/make_rawint4_golden.py
"""
import io
import os
import zipfile

import numpy as np
import torch
from compressed_tensors.compressors.pack_quantized.helpers import pack_to_int32

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rawint4_pack.npz")


def main():
    rng = np.random.default_rng(20261015)
    rows, cols = 4, 512
    q = rng.integers(-8, 8, size=(rows, cols), dtype=np.int8)
    q[0, :16] = np.arange(-8, 8, dtype=np.int8)          # every value at every nibble position of two words
    q[1, :16] = np.arange(7, -9, -1, dtype=np.int8)
    packed = pack_to_int32(torch.from_numpy(q), num_bits=4).numpy()
    assert packed.dtype == np.int32 and packed.shape == (rows, cols // 8)
    scale = torch.from_numpy((rng.random((rows, cols // 32)) * 0.05 + 0.001).astype(np.float32)).to(torch.bfloat16)
    scale_bits = scale.view(torch.int16).numpy().view(np.uint16)
    arrays = {"values": q, "weight_packed": packed, "weight_scale_bits": scale_bits,
              "weight_shape": np.array([rows, cols], dtype=np.int64)}
    with zipfile.ZipFile(OUT, "w", compression=zipfile.ZIP_STORED) as z:
        for name, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(a), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue())
    print("wrote", OUT)


if __name__ == "__main__":
    main()
