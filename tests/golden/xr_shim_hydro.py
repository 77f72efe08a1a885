"""The xarray behaviour the REFERENCE'S OWN hydro path (atlite/hydro.py, convert.py:1087-1149) needs
on top of ``xr_shim.py``, so that ``make_golden_hydro.py`` can run it unmodified.

TEST INFRASTRUCTURE ONLY.  ``xr_shim.DataArray`` is extended by a subclass, installed as the
stand-in ``xarray.DataArray`` for the process that loads hydro.py; the results of every other
generator are untouched.  What it adds, as documented xarray semantics:

  * ``DataArray(series)``: a pandas Series becomes a 1-D array along its index;
  * ``DataArray(values, [(name, index), coordinate, ...])``: coordinates as a list of pairs or
    coordinate arrays;
  * ``sel(dim=label)``: scalar label selection, the dimension dropped;
  * ``roll(dim=n)``: ``np.roll`` along a named dim, coordinates not rolled;
  * ``loc[dict(dim=label)]``: a view of the values, which ``+=`` updates in place.
"""

from __future__ import annotations

import importlib.util
import sys

import numpy as np
import pandas as pd

import xr_shim


class DataArray(xr_shim.DataArray):
    def __init__(self, data=None, coords=None, dims=None, name=None, attrs=None):
        if isinstance(data, pd.Series) and coords is None and dims is None:  # its index is the one dim
            coords, dims = {data.index.name: data.index}, (data.index.name,)
        if isinstance(coords, (list, tuple)) and any(isinstance(c, (tuple, xr_shim.DataArray)) for c in coords):
            pairs = [(c[0], c[1]) if isinstance(c, tuple) else (c.name, c.values) for c in coords]
            dims = dims or tuple(n for n, _ in pairs)
            coords = dict(pairs)
        super().__init__(data, coords, dims, name, attrs)

    # results of arithmetic stay of this class, so that sel / roll / loc remain available
    def _new(self, values, dims=None, coords=None, keep_name=True):
        return DataArray(super()._new(values, dims, coords, keep_name))

    def _bin(self, other, fn, refl=False):
        out = DataArray(super()._bin(other, fn, refl))
        out.name = self.name
        return out

    def _label_view(self, cls, **kw):
        """Scalar label selection: the dims drop out, the values are a VIEW of this array."""
        out = self
        for d, label in kw.items():
            ax = out.dims.index(d)
            i = pd.Index(out._coords[d]).get_loc(label)
            c = {k: v for k, v in out._coords.items() if k != d}
            out = cls(out.values[(slice(None),) * ax + (i,)], c, out.dims[:ax] + out.dims[ax + 1:], out.name)
        return out

    def sel(self, **kw):
        return self._label_view(DataArray, **kw)

    @property
    def loc(self):
        return _Loc(self)

    def roll(self, **shifts):
        v = self.values
        for d, n in shifts.items():
            v = np.roll(v, int(n), axis=self.dims.index(d))
        return self._new(v)


class _Loc:
    def __init__(self, da):
        self.da = da

    def __getitem__(self, key):
        return self.da._label_view(_View, **key)


class _View(DataArray):
    """A label-selected view of another DataArray's values; ``+=`` writes through."""

    def __iadd__(self, other):
        dims, vals, _ = xr_shim._unify((self, other))
        assert tuple(dims) == self.dims, (dims, self.dims)
        self.values += vals[1]
        return self


def load_reference_hydro():
    """atlite/hydro.py from its source file, its imports of shapely and geopandas stood in for, and
    ``atlite.convert`` pointed at it (its ``hydrom``).  Its ``find_basin`` (shapely point-in-polygon)
    and the GeoDataFrame type check are for the caller to replace.  Returns (convert, hydro)."""
    conv = xr_shim.install()
    sys.modules["xarray"].DataArray = DataArray
    geo = xr_shim._module("shapely.geometry", Point=lambda x, y: (x, y))
    xr_shim._module("shapely", geometry=geo)
    spec = importlib.util.spec_from_file_location("atlite.hydro", f"{xr_shim.REF}/hydro.py")
    mod = importlib.util.module_from_spec(spec)
    sys.modules["atlite.hydro"] = mod
    spec.loader.exec_module(mod)
    conv.hydrom = mod
    return conv, mod
