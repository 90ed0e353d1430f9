"""NIfTI-1 (``.nii`` / ``.nii.gz``) reading and writing with the standard library and numpy only: what the test step
(test_2D_fully.py:104-123) does with SimpleITK, which is not a dependency.

* ``read(path)`` -> ``Nifti(array, spacing, header)``: the array in SimpleITK's ``GetArrayFromImage`` order ([z, y, x], x
  fastest), the spacing as SimpleITK's ``GetSpacing`` reports it (``pixdim[1:4]``, i.e. x, y, z) and the parsed 348-byte header
  (either byte order) as a dict of its fields, qform / sform geometry included.
* ``write(path, array, like)`` stores ``array`` as float32 (datatype 16, bitpix 32, ``vox_offset`` 352, magic ``n+1``) with the
  geometry of the header ``like`` (dims, pixdim, ``xyzt_units``, qform / sform codes, quaternion, offsets, srow): the
  ``GetImageFromArray`` + ``CopyInformation`` + ``WriteImage`` sequence of the reference.
* ``header(shape, spacing)`` is a fresh geometry (identity orientation, origin 0) for volumes that have no source file.

The field layout is the NIfTI-1 standard's (nifti1.h).  No file here has been compared with one SimpleITK wrote or read.
"""
import gzip
import struct
from typing import NamedTuple

import numpy as np

# (name, struct code) in file order: the 348-byte nifti_1_header
_FIELDS = (
    ("sizeof_hdr", "i"), ("data_type", "10s"), ("db_name", "18s"), ("extents", "i"), ("session_error", "h"),
    ("regular", "c"), ("dim_info", "B"), ("dim", "8h"), ("intent_p1", "f"), ("intent_p2", "f"), ("intent_p3", "f"),
    ("intent_code", "h"), ("datatype", "h"), ("bitpix", "h"), ("slice_start", "h"), ("pixdim", "8f"), ("vox_offset", "f"),
    ("scl_slope", "f"), ("scl_inter", "f"), ("slice_end", "h"), ("slice_code", "B"), ("xyzt_units", "B"), ("cal_max", "f"),
    ("cal_min", "f"), ("slice_duration", "f"), ("toffset", "f"), ("glmax", "i"), ("glmin", "i"), ("descrip", "80s"),
    ("aux_file", "24s"), ("qform_code", "h"), ("sform_code", "h"), ("quatern_b", "f"), ("quatern_c", "f"), ("quatern_d", "f"),
    ("qoffset_x", "f"), ("qoffset_y", "f"), ("qoffset_z", "f"), ("srow_x", "4f"), ("srow_y", "4f"), ("srow_z", "4f"),
    ("intent_name", "16s"), ("magic", "4s"),
)
_FMT = "".join(code for _, code in _FIELDS)
HEADER_SIZE = 348
assert struct.calcsize("<" + _FMT) == HEADER_SIZE

# fields CopyInformation carries over: size (dims), spacing, origin and direction
GEOMETRY = ("dim", "pixdim", "xyzt_units", "qform_code", "sform_code", "quatern_b", "quatern_c", "quatern_d",
            "qoffset_x", "qoffset_y", "qoffset_z", "srow_x", "srow_y", "srow_z")

# NIfTI-1 datatype code -> numpy dtype (byte order applied at read time)
_DTYPES = {2: "u1", 4: "i2", 8: "i4", 16: "f4", 64: "f8", 256: "i1", 512: "u2", 768: "u4", 1024: "i8", 1280: "u8"}


class Nifti(NamedTuple):
    array: np.ndarray       # [z, y, x] (x fastest), SimpleITK's GetArrayFromImage order
    spacing: tuple          # (x, y, z) = pixdim[1:4], SimpleITK's GetSpacing order
    header: dict


def _open(path, mode):
    return gzip.open(path, mode) if str(path).endswith(".gz") else open(path, mode)


def parse_header(raw):
    """348 bytes (either byte order) -> (dict of the header fields, '<' or '>')"""
    if len(raw) < HEADER_SIZE:
        raise ValueError(f"NIfTI header needs {HEADER_SIZE} bytes, got {len(raw)}")
    for order in "<>":
        if struct.unpack(order + "i", raw[:4])[0] == HEADER_SIZE:
            break
    else:
        raise ValueError("not a NIfTI-1 file: sizeof_hdr is not 348 in either byte order")
    vals = iter(struct.unpack(order + _FMT, raw[:HEADER_SIZE]))
    hdr = {}
    for name, code in _FIELDS:
        n = int(code[:-1]) if code[:-1].isdigit() and not code.endswith("s") else 1
        hdr[name] = tuple(next(vals) for _ in range(n)) if n > 1 else next(vals)
    if hdr["magic"] not in (b"n+1\0", b"ni1\0"):
        raise ValueError(f"not a NIfTI-1 file: magic {hdr['magic']!r}")
    return hdr, order


def pack_header(hdr, order="<"):
    """dict of header fields -> 348 bytes"""
    vals = []
    for name, code in _FIELDS:
        v = hdr[name]
        vals.extend(v if isinstance(v, (tuple, list)) else [v])
    return struct.pack(order + _FMT, *vals)


def _shape_zyx(hdr):
    nd = hdr["dim"][0]
    if not 1 <= nd <= 7:
        raise ValueError(f"NIfTI dim[0] = {nd} is outside 1..7")
    return tuple(int(d) for d in reversed(hdr["dim"][1:nd + 1]))


def read(path):
    """-> Nifti(array [z, y, x], spacing (x, y, z), header).  Stored values are scaled by scl_slope / scl_inter when those are
    set (slope 0 means unscaled), as ITK's reader does."""
    with _open(path, "rb") as f:
        raw = f.read()
    hdr, order = parse_header(raw)
    if hdr["magic"] != b"n+1\0":
        raise ValueError(f"{path}: a two-file NIfTI pair (.hdr/.img) is not supported")
    code = _DTYPES.get(hdr["datatype"])
    if code is None:
        raise ValueError(f"{path}: NIfTI datatype {hdr['datatype']} is not supported")
    shape = _shape_zyx(hdr)
    dt = np.dtype(order + code)
    off, n = int(hdr["vox_offset"]), int(np.prod(shape))
    if len(raw) < off + n * dt.itemsize:
        raise ValueError(f"{path}: {len(raw) - off} data bytes, the header describes {n * dt.itemsize}")
    arr = np.frombuffer(raw, dtype=dt, count=n, offset=off).reshape(shape).astype(dt.newbyteorder("="))
    slope, inter = hdr["scl_slope"], hdr["scl_inter"]
    if slope != 0 and (slope != 1 or inter != 0):
        arr = arr * slope + inter
    return Nifti(arr, tuple(float(v) for v in hdr["pixdim"][1:4]), hdr)


def header(shape, spacing, origin=(0.0, 0.0, 0.0)):
    """A header for a [z, y, x] volume: spacing (x, y, z) in mm, identity orientation at `origin`, qform and sform both set
    (code 1, scanner coordinates)."""
    nz, ny, nx = (int(s) for s in shape)
    sx, sy, sz = (float(s) for s in spacing)
    ox, oy, oz = (float(o) for o in origin)
    hdr = _blank()
    hdr.update(dim=(3, nx, ny, nz, 1, 1, 1, 1), pixdim=(1.0, sx, sy, sz, 0.0, 0.0, 0.0, 0.0), xyzt_units=2 | 8,
               qform_code=1, sform_code=1, quatern_b=0.0, quatern_c=0.0, quatern_d=0.0, qoffset_x=ox, qoffset_y=oy, qoffset_z=oz,
               srow_x=(sx, 0.0, 0.0, ox), srow_y=(0.0, sy, 0.0, oy), srow_z=(0.0, 0.0, sz, oz))
    return hdr


def _blank():
    hdr = {}
    for name, code in _FIELDS:
        if code.endswith("s"):
            hdr[name] = b""
        elif code[:-1].isdigit():
            hdr[name] = (0,) * int(code[:-1])
        else:
            hdr[name] = 0
    hdr.update(sizeof_hdr=HEADER_SIZE, regular=b"r", magic=b"n+1\0")
    return hdr


def write(path, array, like):
    """Write `array` ([z, y, x]) as a float32 single-file NIfTI-1 (gzip-compressed when `path` ends in .gz) carrying the geometry
    of header `like` (CopyInformation: the array must have the size `like` describes)."""
    a = np.ascontiguousarray(array, dtype="<f4")
    if a.shape != _shape_zyx(like):
        raise ValueError(f"array shape {a.shape} differs from the source geometry's {_shape_zyx(like)}")
    hdr = _blank()
    for k in GEOMETRY:
        hdr[k] = like[k]
    hdr.update(datatype=16, bitpix=32, vox_offset=352.0, scl_slope=1.0, scl_inter=0.0)
    data = pack_header(hdr) + b"\0\0\0\0" + a.tobytes()      # 4-byte extension flag: no extensions
    if str(path).endswith(".gz"):
        data = gzip.compress(data, compresslevel=6, mtime=0)     # zlib's default level; mtime 0: same bytes every run
    with open(path, "wb") as f:
        f.write(data)
