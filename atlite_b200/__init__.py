"""atlite_b200 -- H100-native convert+aggregate hot path of PyPSA/atlite.

Drop-in for ``Cutout.convert_and_aggregate`` / ``pv`` / ``wind`` /
``heat_demand`` (reference: atlite/convert.py, atlite/aggregate.py), backed by
hand-written sm_90a CUDA kernels in ``libatlite_b200.so``.
"""

from . import gebco, geotiff, resource, sarah
from ._lib import release_host_staging, set_deterministic
from .convert import (
    coefficient_of_performance,
    convert_and_aggregate,
    convert_coefficient_of_performance,
    convert_cooling_demand,
    convert_csp,
    convert_dewpoint_temperature,
    convert_heat_demand,
    convert_irradiation,
    convert_line_rating,
    convert_many,
    convert_pv,
    convert_runoff,
    convert_soil_temperature,
    convert_solar_thermal,
    convert_temperature,
    convert_wind,
    cooling_demand,
    csp,
    dewpoint_temperature,
    heat_demand,
    irradiation,
    line_rating,
    pv,
    runoff,
    soil_temperature,
    solar_thermal,
    temperature,
    wind,
)
from .cutout import Cutout
from .gis import ExclusionContainer, regrid
from .labelled import DataArray, Dataset, LazyDataset
from .orientation import get_orientation
from .resource import (
    cspinstallations,
    get_cspinstallationconfig,
    get_solarpanelconfig,
    get_windturbineconfig,
    solarpanels,
    windturbine_smooth,
    windturbines,
)

__version__ = "0.1.0"

__all__ = [
    "Cutout", "Dataset", "LazyDataset", "DataArray", "convert_and_aggregate", "convert_many", "convert_pv", "convert_wind",
    "convert_heat_demand", "convert_line_rating", "pv", "wind", "heat_demand", "line_rating", "get_orientation",
    "get_windturbineconfig", "get_solarpanelconfig", "windturbine_smooth", "windturbines",
    "solarpanels", "resource", "set_deterministic", "ExclusionContainer", "regrid",
    "sarah", "gebco", "geotiff",
]
