"""H100-native implementation of the WVA optimizer hot path (see DESIGN.md)."""
from ._abi import ACC_NONE, ACC_UNKNOWN, MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, Allocs  # noqa: F401
from .fleet import Fleet, Grid, config2_grid, synth_fleet  # noqa: F401
from .engine import (Engine, WvaError, accelerator_demand, demand_by_level, greedy_solve,  # noqa: F401,E402
                     slo_envelope, within_margins)
from . import adapters  # noqa: F401,E402
