"""loongcollector_b200 -- H100-native batched log-parsing engine behind LoongCollector's
Processor::Process(PipelineEventGroup&) boundary (see DESIGN.md / INTEGRATION.md).

The product is the C-ABI shared library (include/lc_b200.h); this package is a thin ctypes
binding used by the tests and bench.py.  There is no CPU fallback: loading fails loudly if the
library has not been built, and every compute call fails if no CUDA device is usable."""
from .capi import (Apsara, Engine, HostProcessor, Json, LcError, Regex, Timestamp, device_count, lib, version, LC_ML_IS_LAST,  # noqa: F401
                   LC_ML_MATCHED)
from ._build import build  # noqa: F401
from . import capi  # noqa: F401
