"""amsweep — GPU-native (H100, sm_90a) per-tick HealthCheck schedule-evaluation sweep.

Drop-in for ONE hot path of keikoproj/active-monitor: the schedule ladder and
remedy state machine of internal/controllers/healthcheck_controller.go
(:225-267, :633-724, :819-852, :745-752), re-expressed as a batch sweep over
SoA records in HBM behind a C-ABI (include/amsweep.h).

The package directory is ``active-monitor_b200`` (not an identifier): import it
with ``importlib.import_module("active-monitor_b200")``.
"""
from . import _lib as abi  # noqa: F401
from ._lib import *  # noqa: F401,F403  (constants + ctypes structs)
from .sweep import (AmError, Cron, CronParseError, CronUnsupported, Sweep, alloc_columns,  # noqa: F401
                    checkpoint_delta_info, checkpoint_info, civil_from_unix, classify, cols_struct, columns_to_records, cron_parse,
                    records_to_columns, remedy_is_empty, tz_lookup, tz_offset)


def load():
    """dlopen libamsweep.so (raises ImportError when it has not been built)."""
    return abi.load()
