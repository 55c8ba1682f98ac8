"""xarray when it is installed, otherwise a small DataArray with the subset of the xarray API
that the rollout path uses (the reference returns ``xr.DataArray(dims=time,channel,lat,lon)``
from /root/reference/skyrim/core/models/utils.py:42-49 and consumes it in
``GlobalPrediction`` base.py:149-274 and ``save_forecast`` common.py:115-204).

The build / bench image has no xarray, zarr or netCDF4; scipy's netCDF3 writer is available.
"""
from __future__ import annotations

import json
import os
from pathlib import Path

import numpy as np

try:  # pragma: no cover - exercised only where xarray exists
    import xarray as _xr
    HAVE_XARRAY = True
except Exception:  # noqa: BLE001
    _xr = None
    HAVE_XARRAY = False


def _as_index(values, key, method=None):
    vals = np.asarray(values)
    if isinstance(key, slice):
        if key.start is None and key.stop is None:
            return slice(None)
        lo = key.start if key.start is not None else vals.min()
        hi = key.stop if key.stop is not None else vals.max()
        a, b = (lo, hi) if lo <= hi else (hi, lo)
        return np.nonzero((vals >= a) & (vals <= b))[0]
    if isinstance(key, (list, tuple, np.ndarray)):
        return np.array([_as_index(values, k, method) for k in key])
    if vals.dtype.kind in "fiu" and not isinstance(key, str):
        if method == "nearest":
            return int(np.abs(vals.astype(np.float64) - float(key)).argmin())
        hit = np.nonzero(vals == key)[0]
    else:
        hit = np.nonzero(vals == key)[0]
    if hit.size == 0:
        raise KeyError(key)
    return int(hit[0])


class DataArray:
    """Minimal stand-in for xarray.DataArray (values + named dims + 1-D coords).  A coordinate that is not a dimension may
    lie along one, given as ``(dim, values)`` as xarray takes it (a site's lat / lon along "site"); ``coords[name]`` is
    then its values, and selecting along the dimension selects them too."""

    def __init__(self, data, dims, coords=None, name=None, attrs=None):
        self.values = np.asarray(data)
        self.dims = tuple(dims)
        assert self.values.ndim == len(self.dims), (self.values.shape, dims)
        self.coords = {}
        self.coord_dims = {}   # non-dimension coordinate -> the dimension it lies along
        for k, v in (coords or {}).items():
            if isinstance(v, tuple) and len(v) == 2 and v[0] in self.dims and k not in self.dims:
                self.coord_dims[k], v = v[0], np.asarray(v[1])
                assert v.shape == (self.values.shape[self.dims.index(self.coord_dims[k])],), (k, v.shape, self.values.shape)
            elif k in self.dims:
                v = np.asarray(v)
                assert v.shape[0] == self.values.shape[self.dims.index(k)], (k, v.shape, self.values.shape)
            self.coords[k] = v
        self.name = name
        self.attrs = dict(attrs or {})

    # -- basic protocol --------------------------------------------------------------------
    @property
    def shape(self):
        return self.values.shape

    @property
    def size(self):
        return self.values.size

    @property
    def dtype(self):
        return self.values.dtype

    def __getattr__(self, item):  # da.lat / da.channel / da.time
        coords = self.__dict__.get("coords", {})
        if item in coords:
            return DataArray(np.asarray(coords[item]), (item,), {item: coords[item]})
        raise AttributeError(item)

    def __contains__(self, x):
        return x in self.values

    def __repr__(self):
        return f"<DataArray {dict(zip(self.dims, self.shape))} {self.values.dtype}>"

    def item(self):
        return self.values.item()

    def _take(self, dim, idx):
        ax = self.dims.index(dim)
        vals = np.take(self.values, idx, axis=ax) if not isinstance(idx, slice) else self.values[(slice(None),) * ax + (idx,)]
        coords = dict(self.coords)
        dims = list(self.dims)
        along = self.__dict__.get("coord_dims", {})
        for k in [dim] + [k for k, d in along.items() if d == dim]:
            if k in coords:
                coords[k] = np.asarray(coords[k])[idx]
        if isinstance(idx, (int, np.integer)):
            dims.pop(ax)
        else:   # the non-dimension coordinates keep their dimension
            coords.update({k: (d, coords[k]) for k, d in along.items() if d == dim})
        coords.update({k: (d, coords[k]) for k, d in along.items() if d != dim})
        return DataArray(vals, dims, coords, self.name, self.attrs)

    def isel(self, **kw):
        out = self
        for dim, idx in kw.items():
            out = out._take(dim, idx)
        return out

    def sel(self, method=None, **kw):
        out = self
        for dim, key in kw.items():
            out = out._take(dim, _as_index(out.coords[dim], key, method))
        return out

    def squeeze(self):
        out = self
        for dim, n in list(zip(self.dims, self.shape)):
            if n == 1:
                out = out._take(dim, 0)
        return out

    def __getitem__(self, key):
        if isinstance(key, (list, tuple)) and key and isinstance(key[0], str):
            return self.sel(channel=list(key))  # pred[filter_vars] in save_forecast (common.py:132)
        return DataArray(self.values[key], self.dims, self.coords) if key is Ellipsis else self.isel(**{self.dims[0]: key})

    # -- persistence ------------------------------------------------------------------------
    def to_netcdf(self, path, engine="scipy"):
        from scipy.io import netcdf_file
        with netcdf_file(os.fspath(path), "w", version=2) as f:
            for d, n in zip(self.dims, self.shape):
                f.createDimension(d, n)
            for d in self.dims:
                c = self.coords.get(d)
                if c is None:
                    continue
                c = np.asarray(c)
                if d == "time":
                    v = f.createVariable(d, "d", (d,))
                    v[:] = np.array([np.datetime64(t, "s").astype("int64") for t in c], dtype=np.float64)
                    v.units = b"seconds since 1970-01-01 00:00:00"
                elif c.dtype.kind in "US":
                    width = max(len(str(s)) for s in c)
                    f.createDimension(f"{d}_strlen", width)
                    v = f.createVariable(d, "c", (d, f"{d}_strlen"))
                    v[:] = np.array([list(str(s).ljust(width)) for s in c], dtype="S1")
                else:
                    v = f.createVariable(d, "d", (d,))
                    v[:] = c.astype(np.float64)
            wide = self.values.dtype == np.float64   # fp64 arrays (scorecards) keep their precision; the rest is fp32
            var = f.createVariable(self.name or "__xarray_dataarray_variable__", "d" if wide else "f", self.dims)
            var[:] = self.values.astype(np.float64 if wide else np.float32)
            along = self.__dict__.get("coord_dims", {})
            if along:   # after the data variable, named by its CF "coordinates" attribute, as xarray writes them
                var.coordinates = " ".join(along).encode()
                for k, d in along.items():
                    v = f.createVariable(k, "d", (d,))
                    v[:] = np.asarray(self.coords[k]).astype(np.float64)
            for k, v in self.attrs.items():   # scalar attributes become global attributes, as xarray writes them
                setattr(f, k, v)

    def to_zarr(self, store, mode="w", append_dim=None, consolidated=True):
        """zarr v2 directory store, uncompressed, one chunk per leading index."""
        root = Path(store)
        name = self.name or "__xarray_dataarray_variable__"
        if mode == "a" and root.exists() and append_dim:
            meta = json.loads((root / name / ".zarray").read_text())
            ax = self.dims.index(append_dim)
            assert ax == 0, "append along the leading dimension only"
            n0 = meta["shape"][0]
            meta["shape"][0] = n0 + self.shape[0]
            for i in range(self.shape[0]):
                _write_chunk(root / name, (n0 + i,) + (0,) * (self.values.ndim - 1), self.values[i:i + 1].astype("<f4"))
            (root / name / ".zarray").write_text(json.dumps(meta))
            cmeta = json.loads((root / append_dim / ".zarray").read_text())
            old = np.frombuffer((root / append_dim / "0").read_bytes(), dtype=cmeta["dtype"])
            new = np.concatenate([old, _encode_coord(self.coords[append_dim])[0]])
            cmeta["shape"] = [int(new.shape[0])]
            cmeta["chunks"] = [int(new.shape[0])]
            (root / append_dim / "0").write_bytes(new.tobytes())
            (root / append_dim / ".zarray").write_text(json.dumps(cmeta))
        else:
            root.mkdir(parents=True, exist_ok=True)
            (root / ".zgroup").write_text(json.dumps({"zarr_format": 2}))
            (root / ".zattrs").write_text("{}")
            _write_array(root / name, self.values.astype("<f4"), (1,) + self.shape[1:], list(self.dims))
            for d in self.dims:
                if d in self.coords:
                    enc, attrs = _encode_coord(self.coords[d])
                    _write_array(root / d, enc, enc.shape, [d], attrs)
        if consolidated:
            md = {}
            for p in sorted(root.rglob(".z*")):
                if p.name != ".zmetadata":
                    md[p.relative_to(root).as_posix()] = json.loads(p.read_text())
            (root / ".zmetadata").write_text(json.dumps({"zarr_consolidated_format": 1, "metadata": md}))


def _encode_coord(c):
    c = np.asarray(c)
    if c.dtype.kind == "M" or (c.dtype == object and len(c) and hasattr(c[0], "year")):
        return np.array([np.datetime64(t, "s").astype("int64") for t in c], dtype="<i8"), {
            "units": "seconds since 1970-01-01 00:00:00", "calendar": "proleptic_gregorian"}
    if c.dtype.kind in "US" or c.dtype == object:
        w = max(len(str(s)) for s in c)
        return np.array([str(s) for s in c], dtype=f"<U{w}"), {}
    return c.astype("<f8"), {}


def _write_chunk(path: Path, idx, block):
    (path / ".".join(str(i) for i in idx)).write_bytes(np.ascontiguousarray(block).tobytes())


def _write_array(path: Path, arr, chunks, dims, attrs=None):
    path.mkdir(parents=True, exist_ok=True)
    meta = {"zarr_format": 2, "shape": list(arr.shape), "chunks": list(chunks), "dtype": arr.dtype.str,
            "compressor": None, "fill_value": None, "order": "C", "filters": None}
    (path / ".zarray").write_text(json.dumps(meta))
    (path / ".zattrs").write_text(json.dumps({"_ARRAY_DIMENSIONS": dims, **(attrs or {})}))
    if arr.ndim == 1 or tuple(chunks) == tuple(arr.shape):
        _write_chunk(path, (0,) * arr.ndim, arr)
    else:
        for i in range(arr.shape[0]):
            _write_chunk(path, (i,) + (0,) * (arr.ndim - 1), arr[i:i + 1])


def _attr(var, key):
    v = getattr(var, key, b"")
    return v.decode() if isinstance(v, bytes) else str(v)


def open_dataarray(path, engine=None):
    """netCDF3 file or zarr v2 directory written by the methods above."""
    p = Path(path)
    if p.is_dir():
        md = json.loads((p / ".zmetadata").read_text())["metadata"] if (p / ".zmetadata").exists() else None
        name = "__xarray_dataarray_variable__"
        meta = json.loads((p / name / ".zarray").read_text())
        dims = json.loads((p / name / ".zattrs").read_text())["_ARRAY_DIMENSIONS"]
        shape = meta["shape"]
        data = np.empty(shape, dtype=meta["dtype"])
        for i in range(shape[0]):
            blk = np.frombuffer((p / name / ".".join([str(i)] + ["0"] * (len(shape) - 1))).read_bytes(), dtype=meta["dtype"])
            data[i] = blk.reshape(shape[1:])
        coords = {}
        for d in dims:
            if (p / d / ".zarray").exists():
                cm = json.loads((p / d / ".zarray").read_text())
                c = np.frombuffer((p / d / "0").read_bytes(), dtype=cm["dtype"])
                if d == "time":
                    c = c.astype("datetime64[s]")
                coords[d] = c
        del md
        return DataArray(data, dims, coords)
    from scipy.io import netcdf_file
    with netcdf_file(os.fspath(p), "r", mmap=False) as f:
        names = [k for k in f.variables if k not in f.dimensions]
        aux = list(dict.fromkeys(c for k in names for c in _attr(f.variables[k], "coordinates").split()))
        name = [k for k in names if k not in aux][0]
        var = f.variables[name]
        dims = list(var.dimensions)
        coords = {c: (f.variables[c].dimensions[0], np.array(f.variables[c][:], dtype=np.float64)) for c in aux
                  if c in f.variables}
        for d in dims:
            if d in f.variables:
                v = f.variables[d]
                if v.typecode() == "c":
                    coords[d] = np.array(["".join(ch.decode() for ch in row).strip() for row in v[:]])
                elif d == "time":
                    coords[d] = np.asarray(v[:]).astype("int64").astype("datetime64[s]")
                else:
                    coords[d] = np.array(v[:])
        attrs = {k: v.decode() if isinstance(v, bytes) else v.item() if np.ndim(v) == 0 or np.size(v) == 1 else v
                 for k, v in f._attributes.items()}
        return DataArray(np.array(var[:]), dims, coords, attrs=attrs)


if HAVE_XARRAY:  # pragma: no cover
    DataArray = _xr.DataArray  # noqa: F811
    open_dataarray = _xr.open_dataarray  # noqa: F811
