"""Counterpart of ``open3d.utility`` on this path: the library's global random engine (``random``)."""
from . import random  # noqa: F401
