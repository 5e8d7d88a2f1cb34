"""mrbayes_b200 -- H100-native tree-likelihood engine for MrBayes.

The product is the CUDA shared library ``mrbayes_b200/lib/libmb200.so`` (C-ABI:
``include/mb200.h``) plus the C seam ``mrbayes_b200/seam/`` that plugs it into MrBayes'
``LaunchLogLikeForDivision`` call site.  This Python package is tooling around it:
ctypes bindings (``abi``), evaluation-record I/O (``records``) and synthetic workload
generators (``workloads``) for tests and ``bench.py``.
"""
__version__ = "0.1.0"
