"""lepton_b200 -- H100 (sm_90a) implementation of Lepton's arithmetic-coding hot path.

The product is the C-ABI shared library ``lepton_b200/liblepton_b200.so`` (hand-written sm_90a CUDA kernels +
C++ host code, built by ``__graft_entry__.build()`` / ``lepton_b200/build.py``); this package is the thin Python
mirror of the reference's codec surface used by the tests and the benchmark.  There is no CPU fallback: importing
works anywhere, but creating a codec without the built library or without a CUDA device raises.
"""
from .codec import (CODER_ANS, CODER_BOOL, CoefImage, HostJpeg, HostLep, LeptonB200Codec, LeptonB200Error, LeptonB200FileCodec, LeptonB200MultiGpuFileCodec, lep_members, lib, shard_by_size_native,  # noqa: F401
                    library_path)
