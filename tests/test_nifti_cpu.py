"""NIfTI-1 reader / writer (wsl4mis_b200/nifti.py) against the layout of the NIfTI-1 standard (nifti1.h): header fields at their
byte offsets, both byte orders, .nii and .nii.gz, and the geometry a written file takes from its source header."""
import gzip
import struct

import numpy as np
import pytest

from wsl4mis_b200 import nifti

# nifti1.h: (offset, struct code) of the fields the writer sets or copies
OFFSETS = {
    "sizeof_hdr": (0, "i"), "dim": (40, "8h"), "datatype": (70, "h"), "bitpix": (72, "h"), "pixdim": (76, "8f"),
    "vox_offset": (108, "f"), "scl_slope": (112, "f"), "scl_inter": (116, "f"), "xyzt_units": (123, "B"),
    "qform_code": (252, "h"), "sform_code": (254, "h"), "quatern_b": (256, "f"), "quatern_c": (260, "f"), "quatern_d": (264, "f"),
    "qoffset_x": (268, "f"), "qoffset_y": (272, "f"), "qoffset_z": (276, "f"), "srow_x": (280, "4f"), "srow_y": (296, "4f"),
    "srow_z": (312, "4f"), "magic": (344, "4s"),
}


def _source(shape=(5, 7, 9)):
    """a header with an oblique orientation, an offset origin and anisotropic spacing, as a scanner file has"""
    h = nifti.header(shape, (1.37, 1.25, 6.5), origin=(-120.5, 88.25, -30.0))
    h.update(quatern_b=0.1, quatern_c=-0.2, quatern_d=0.3, pixdim=(-1.0,) + h["pixdim"][1:], sform_code=2,
             srow_x=(1.3, 0.1, 0.2, -120.5), srow_y=(-0.1, 1.2, 0.3, 88.25), srow_z=(0.05, -0.2, 6.4, -30.0))
    return h


def _values(raw, name, order="<"):
    off, code = OFFSETS[name]
    v = struct.unpack_from(order + code, raw, off)
    return v if len(v) > 1 else v[0]


@pytest.mark.parametrize("ext", [".nii", ".nii.gz"])
def test_written_header_matches_the_nifti1_layout(tmp_path, ext):
    a = np.random.RandomState(0).rand(5, 7, 9).astype(np.float64) * 100
    src = _source()
    path = str(tmp_path / ("v" + ext))
    nifti.write(path, a, src)
    raw = open(path, "rb").read()
    if ext == ".nii.gz":
        assert raw[:2] == b"\x1f\x8b"
        raw = gzip.decompress(raw)
    else:
        assert raw[:4] == struct.pack("<i", 348)
    assert _values(raw, "sizeof_hdr") == 348
    assert _values(raw, "dim") == (3, 9, 7, 5, 1, 1, 1, 1)           # x, y, z
    assert _values(raw, "datatype") == 16 and _values(raw, "bitpix") == 32
    assert _values(raw, "vox_offset") == 352.0
    assert _values(raw, "scl_slope") == 1.0 and _values(raw, "scl_inter") == 0.0
    assert _values(raw, "magic") == b"n+1\0"
    for name in ("pixdim", "xyzt_units", "qform_code", "sform_code", "quatern_b", "quatern_c", "quatern_d", "qoffset_x",
                 "qoffset_y", "qoffset_z", "srow_x", "srow_y", "srow_z"):
        want = src[name]
        want = tuple(np.float32(w) for w in want) if isinstance(want, tuple) else (np.float32(want) if isinstance(want, float) else want)
        assert _values(raw, name) == want, name
    assert raw[348:352] == b"\0\0\0\0"                                   # no extensions
    assert len(raw) == 352 + a.size * 4
    data = np.frombuffer(raw, "<f4", offset=352).reshape(9 * 7 * 5)
    assert np.array_equal(data, a.astype(np.float32).ravel())          # x fastest: C order of [z, y, x]


@pytest.mark.parametrize("ext", [".nii", ".nii.gz"])
def test_round_trip_keeps_data_spacing_and_geometry(tmp_path, ext):
    a = np.random.RandomState(1).randint(0, 4, size=(5, 7, 9)).astype(np.float32)
    src = _source()
    path = str(tmp_path / ("v" + ext))
    nifti.write(path, a, src)
    got = nifti.read(path)
    assert got.array.dtype == np.float32 and got.array.shape == (5, 7, 9)
    assert np.array_equal(got.array, a)
    assert got.spacing == tuple(float(np.float32(s)) for s in (1.37, 1.25, 6.5))
    for name in nifti.GEOMETRY:
        v = src[name]
        want = tuple(float(np.float32(x)) for x in v) if name in ("pixdim", "srow_x", "srow_y", "srow_z") else v
        if isinstance(v, float):
            want = float(np.float32(v))
        assert got.header[name] == want, name
    # a file written from a read header carries the same geometry again
    path2 = str(tmp_path / ("w" + ext))
    nifti.write(path2, got.array * 2, got.header)
    again = nifti.read(path2)
    assert all(again.header[k] == got.header[k] for k in nifti.GEOMETRY)
    assert np.array_equal(again.array, a * 2)


def _hand_written(path, order, arr, code, bitpix, slope=0.0, inter=0.0):
    """a single-file NIfTI-1 in byte order `order` built field by field from the spec's offsets"""
    nz, ny, nx = arr.shape
    raw = bytearray(352)
    struct.pack_into(order + "i", raw, 0, 348)
    struct.pack_into(order + "8h", raw, 40, 3, nx, ny, nz, 1, 1, 1, 1)
    struct.pack_into(order + "hh", raw, 70, code, bitpix)
    struct.pack_into(order + "8f", raw, 76, 1.0, 1.5625, 1.25, 10.0, 0, 0, 0, 0)
    struct.pack_into(order + "fff", raw, 108, 352.0, slope, inter)
    struct.pack_into(order + "hh", raw, 252, 1, 1)
    struct.pack_into(order + "12f", raw, 280, 1.5625, 0, 0, 1, 0, 1.25, 0, 2, 0, 0, 10.0, 3)
    struct.pack_into("4s", raw, 344, b"n+1\0")
    data = bytes(raw) + arr.astype(arr.dtype.newbyteorder(order)).tobytes()
    with (gzip.open(path, "wb") if path.endswith(".gz") else open(path, "wb")) as f:
        f.write(data)


@pytest.mark.parametrize("ext", [".nii", ".nii.gz"])
@pytest.mark.parametrize("dtype,code,bitpix", [(np.int16, 4, 16), (np.uint8, 2, 8), (np.float32, 16, 32), (np.float64, 64, 64)])
def test_reads_both_byte_orders(tmp_path, ext, dtype, code, bitpix):
    arr = (np.arange(3 * 4 * 5).reshape(3, 4, 5) % 200).astype(dtype)
    out = {}
    for order in "<>":
        path = str(tmp_path / f"{'le' if order == '<' else 'be'}{ext}")
        _hand_written(path, order, arr, code, bitpix)
        out[order] = nifti.read(path)
    for r in out.values():
        assert r.array.shape == (3, 4, 5) and np.array_equal(r.array, arr)
        assert r.spacing == (1.5625, 1.25, 10.0)
        assert r.header["qform_code"] == 1 and r.header["srow_y"] == (0.0, 1.25, 0.0, 2.0)
    assert all(out["<"].header[k] == out[">"].header[k] for k in nifti.GEOMETRY)


def test_scaling_and_bad_input(tmp_path):
    arr = np.arange(24, dtype=np.int16).reshape(2, 3, 4)
    p = str(tmp_path / "s.nii")
    _hand_written(p, "<", arr, 4, 16, slope=0.5, inter=-1.0)
    assert np.array_equal(nifti.read(p).array, arr * 0.5 - 1.0)
    with pytest.raises(ValueError, match="differs from the source geometry"):
        nifti.write(str(tmp_path / "x.nii"), np.zeros((2, 3, 5)), nifti.read(p).header)
    open(str(tmp_path / "bad.nii"), "wb").write(b"\0" * 400)
    with pytest.raises(ValueError, match="sizeof_hdr"):
        nifti.read(str(tmp_path / "bad.nii"))
