"""CPU tests of the GLB export (perf_b200.mesh.write_glb / read_glb): the size limit as a pure function of the counts, and an
untextured mesh written and read back -- the GLB header and chunk layout, 4-byte alignment, every accessor inside its
bufferView, POSITION's min / max, indices below the vertex count, and the data back exactly (colours through linear fp32)."""
import json
import struct

import numpy as np
import pytest

from perf_b200 import mesh as M


def test_size_limit_is_a_function_of_counts():
    # the per-face atlas at 16384^2: 33.5 M faces split into 100.7 M vertices of position, normal, uv and tangent (48 B each)
    F = 33_554_432
    with pytest.raises(ValueError, match="2\\^32 - 1"):
        M.check_glb_size(3 * F, 0, True, False, True, True)
    assert M.glb_bytes(3 * F, 0, True, False, True, True) > 4.8e9
    M.check_glb_size(3_000_000, 0, True, False, True, True, [50_000_000, 60_000_000])
    # the bound grows by exactly the data written per vertex and index
    base = M.glb_bytes(0, 0, True, True, False, False)
    assert M.glb_bytes(10, 30, True, True, False, False) - base == 10 * 36 + 30 * 4
    assert M.glb_bytes(0, 0, False, False, False, False, [5]) - M.glb_bytes(0, 0, False, False, False, False) == 8


def _mesh(seed=0, V=500, F=900):
    g = np.random.default_rng(seed)
    n = g.normal(size=(V, 3)).astype(np.float32)
    return {"vertices": (g.random((V, 3)) * 4 - 2).astype(np.float32), "faces": g.integers(0, V, (F, 3)).astype(np.int32),
            "normals": n / np.linalg.norm(n, axis=1, keepdims=True), "colors": g.integers(0, 256, (V, 3)).astype(np.uint8)}


def test_untextured_roundtrip(tmp_path):
    m = _mesh()
    m["colors"][:256, 0] = np.arange(256)                    # every byte value through linear fp32 and back
    path = str(tmp_path / "m.glb")
    M.write_glb(path, m)
    data = open(path, "rb").read()
    magic, version, total = struct.unpack_from("<III", data, 0)
    assert (magic, version, total) == (0x46546C67, 2, len(data))
    jl, jt = struct.unpack_from("<II", data, 12)
    assert jt == 0x4E4F534A and jl % 4 == 0 and data[20 + jl - 1:20 + jl] in (b"}", b" ")
    doc = json.loads(data[20:20 + jl])
    bl, bt = struct.unpack_from("<II", data, 20 + jl)
    assert bt == 0x004E4942 and bl % 4 == 0 and 28 + jl + bl == len(data) and doc["buffers"][0]["byteLength"] == bl
    for v in doc["bufferViews"]:
        assert v["byteOffset"] % 4 == 0 and v["byteOffset"] + v["byteLength"] <= bl
    size = {5126: 4, 5125: 4}
    comps = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4}
    for a in doc["accessors"]:
        v = doc["bufferViews"][a["bufferView"]]
        assert a["count"] * comps[a["type"]] * size[a["componentType"]] <= v["byteLength"]
    prim = doc["meshes"][0]["primitives"][0]
    assert set(prim["attributes"]) == {"POSITION", "NORMAL", "COLOR_0"} and prim["mode"] == 4
    pos = doc["accessors"][prim["attributes"]["POSITION"]]
    assert pos["min"] == [float(x) for x in m["vertices"].min(0)] and pos["max"] == [float(x) for x in m["vertices"].max(0)]
    mat = doc["materials"][prim["material"]]
    assert "KHR_materials_unlit" in mat["extensions"] and doc["extensionsUsed"] == ["KHR_materials_unlit"]
    assert mat["doubleSided"] is False
    q = doc["nodes"][0]["rotation"]
    assert q == [-np.sqrt(0.5), 0.0, 0.0, np.sqrt(0.5)]

    r = M.read_glb(path)
    assert int(r["faces"].max()) < r["vertices"].shape[0]
    for k in ("vertices", "faces", "normals", "colors"):
        assert np.array_equal(r[k], m[k]), k
    lin = np.frombuffer(data, np.float32, count=3 * 500, offset=28 + jl + doc["bufferViews"][
        doc["accessors"][prim["attributes"]["COLOR_0"]]["bufferView"]]["byteOffset"]).reshape(-1, 3)
    assert lin.min() >= 0 and lin.max() <= 1 and lin[255, 0] == 1.0 and lin[0, 0] == 0.0
    assert np.all(np.diff(lin[:256, 0]) > 0)


def test_untextured_without_colors_or_normals(tmp_path):
    m = _mesh(1)
    del m["colors"], m["normals"]
    path = str(tmp_path / "m.glb")
    M.write_glb(path, m)
    r = M.read_glb(path)
    assert set(r["gltf"]["meshes"][0]["primitives"][0]["attributes"]) == {"POSITION"}
    assert np.array_equal(r["vertices"], m["vertices"]) and np.array_equal(r["faces"], m["faces"])
