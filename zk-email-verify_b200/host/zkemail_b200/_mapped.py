"""(pointer, length) of a file image for the C ABI, shared by the `.ptau` and `.r1cs` readers."""
from __future__ import annotations
import ctypes


class mapped_buffer:
    """(pointer, length) of a file image given as bytes, a buffer or a path; a path is memory-mapped copy-on-write (a `.ptau`
    for a large domain is several GB, a circom EmailVerifier `.r1cs` up to about 1 GB), so nothing is read that the library
    does not touch."""

    def __init__(self, src):
        self._src, self._mm, self._arr = src, None, None

    def __enter__(self):
        import mmap
        import os
        p = self._src
        if isinstance(p, (str, os.PathLike)):
            with open(p, "rb") as f:
                self._mm = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_COPY)
            p = self._mm
        if isinstance(p, bytes):
            return p, len(p)
        with memoryview(p) as mv:
            if mv.readonly:
                return bytes(mv), mv.nbytes
            n = mv.nbytes
        self._arr = (ctypes.c_char * n).from_buffer(p)
        return ctypes.addressof(self._arr), n

    def __exit__(self, *exc):
        self._arr = None
        if self._mm is not None:
            self._mm.close()
        return False
