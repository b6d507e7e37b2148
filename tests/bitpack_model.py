"""Which kernel pack_bits (csrc/bitpack.cuh) runs to build a bit volume: the restatement that the path
tests of flood fill and marching cubes check their case lists against."""
import numpy as np

VEC = ("vec<uint8,linear>", "vec<uint8,rows>", "vec<int16,linear>", "vec<int16,rows>")
BALLOT = ("ballot<uint8>", "ballot<int16>")


def pack_kernel(dtype, dx, data_offset=0, other_offset=None):
    """The packing kernel for [..][dx] rows of int16 or uint8 data whose device pointer lies data_offset
    bytes past a 16-byte boundary, with a uint8 `other` stream other_offset bytes past one (None: no
    stream). Empty ranges launch neither: the launcher clears the bits instead."""
    dtype = np.dtype(dtype)
    group = 16 // dtype.itemsize                  # voxels per 128-bit load; the stream loads as many bytes
    if dx % group == 0 and data_offset % 16 == 0 and (other_offset is None or other_offset % group == 0):
        return f"vec<{dtype.name},{'linear' if dx % 32 == 0 else 'rows'}>"
    return f"ballot<{dtype.name}>"
