"""comet_b200 -- Python host side of the H100-native hot path of apache/datafusion-comet.

`native` binds the C ABI (libcomet_b200.so), `proto` encodes the reference's plan IR and `tpch`
holds the benchmark plans / data.  All compute happens in the shared library's CUDA kernels.
"""
from . import native, proto, tpch  # noqa: F401
