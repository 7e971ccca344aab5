"""persia_b200 — PERSIA's sparse-embedding hot path on H100 (sm_90a), behind a C ABI.

See DESIGN.md.  The product path is libpersia_b200.so (persia_b200/csrc); this package only binds it
(native.py), owns device buffers through torch (shard.py) and mirrors the reference's host interface.
"""
from . import native  # noqa: F401

__all__ = ["native"]
__version__ = "0.1.0"
