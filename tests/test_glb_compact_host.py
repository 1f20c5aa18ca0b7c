"""CPU tests of the compact GLB (perf_b200.mesh.write_glb(compact=True) / read_glb) on an untextured mesh: the
KHR_mesh_quantization layout (declared used and required, byte strides, normalised integer accessors), the node transform
that undoes the position quantisation, and the data read back within the quantisation bounds (positions within half a step
per axis, normals within int8 rounding, colours exact); and the size bound of the compact layout."""
import json
import struct

import numpy as np

from perf_b200 import mesh as M

from test_glb_host import _mesh


def test_compact_size_is_a_function_of_counts():
    base = M.glb_bytes(0, 0, True, True, False, False, compact=True)
    assert M.glb_bytes(10, 30, True, True, False, False, compact=True) - base == 10 * 20 + 30 * 4
    # per-face atlas with a normal texture 48 -> 24 bytes per vertex, chart atlas 32 -> 20
    assert M.glb_bytes(1, 0, True, False, True, True, compact=True) - M.glb_bytes(0, 0, True, False, True, True, compact=True) == 24
    assert M.glb_bytes(1, 0, True, False, True, False, compact=True) - M.glb_bytes(0, 0, True, False, True, False, compact=True) == 20
    F = 33_554_432
    M.check_glb_size(3 * F, 0, True, False, True, True, compact=True)        # 2.4 GB: fits where the exact layout does not


def _quat_matrix(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


# The angle between a unit vector and its int8 code decoded (c / 127): the error vector has at most 0.5 / 127 per component
INT8_ANGLE = float(np.arcsin(np.sqrt(3) * 0.5 / 127))


def test_untextured_compact_roundtrip(tmp_path):
    """A mesh in a box of the proportions of a room (1.2 x 1.6 x 0.9), so that a per-axis scale would show: positions within
    half a step (the largest extent / 65535) per axis, colours exact, normals within int8 rounding -- read back and as a
    glTF viewer sees them through the node's normal matrix."""
    m = _mesh(2)
    m["vertices"] = (m["vertices"] * np.array([0.3, 0.4, 0.225], np.float32)).astype(np.float32)
    m["colors"][:256, 1] = np.arange(256)
    path = str(tmp_path / "m.glb")
    M.write_glb(path, m, compact=True)
    data = open(path, "rb").read()
    jl, _ = struct.unpack_from("<II", data, 12)
    doc = json.loads(data[20:20 + jl])
    assert doc["extensionsRequired"] == ["KHR_mesh_quantization"]
    assert doc["extensionsUsed"] == ["KHR_materials_unlit", "KHR_mesh_quantization"]
    prim = doc["meshes"][0]["primitives"][0]
    acc = {k: doc["accessors"][i] for k, i in prim["attributes"].items()}
    want = {"POSITION": (5123, 8), "NORMAL": (5120, 4), "COLOR_0": (5123, 8)}
    assert set(acc) == set(want)
    for k, (ct, stride) in want.items():
        v = doc["bufferViews"][acc[k]["bufferView"]]
        assert acc[k]["componentType"] == ct and acc[k]["normalized"] is True and acc[k]["type"] == "VEC3"
        assert v["byteStride"] == stride and v["byteLength"] == stride * acc[k]["count"] and v["byteOffset"] % 4 == 0
    node = doc["nodes"][0]
    lo, hi = m["vertices"].min(0).astype(np.float64), m["vertices"].max(0).astype(np.float64)
    ext = float((hi - lo).max())
    assert acc["POSITION"]["min"] == [0, 0, 0] and max(acc["POSITION"]["max"]) == 65535
    assert node["scale"] == [ext] * 3 and node["rotation"] == [-np.sqrt(0.5), 0.0, 0.0, np.sqrt(0.5)]
    assert node["translation"] == [float(lo[0]), float(lo[2]), float(-lo[1])]

    # the node's M = T R S applied to the normalised positions gives the world positions rotated to +Y up
    R = _quat_matrix(node["rotation"])
    base = 28 + jl
    v0 = doc["bufferViews"][acc["POSITION"]["bufferView"]]
    q = np.frombuffer(data, np.uint16, count=4 * 500, offset=base + v0["byteOffset"]).reshape(-1, 4)[:, :3] / 65535.0
    gl = (q * np.asarray(node["scale"])) @ R.T + np.asarray(node["translation"])
    w = m["vertices"].astype(np.float64)
    step = ext / 65535
    assert np.all(np.abs(gl - w @ R.T) <= 0.5 * step * (1 + 1e-6) + 1e-7)

    # what a viewer shades with: the stored normal through the inverse transpose of R S, normalised, against the world
    # normal rotated +Z -> +Y
    v1 = doc["bufferViews"][acc["NORMAL"]["bufferView"]]
    n8 = np.frombuffer(data, np.int8, count=4 * 500, offset=base + v1["byteOffset"]).reshape(-1, 4)[:, :3]
    n = np.maximum(n8 / 127.0, -1.0) @ np.linalg.inv(R @ np.diag(node["scale"]))   # row vectors: n (RS)^-1 = ((RS)^-T n)^T
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    ang = np.arccos(np.clip((n * (m["normals"].astype(np.float64) @ R.T)).sum(1), -1, 1))
    assert ang.max() <= INT8_ANGLE + 1e-6, np.degrees(ang.max())

    r = M.read_glb(path)
    assert np.array_equal(r["faces"], m["faces"]) and np.array_equal(r["colors"], m["colors"])
    assert r["vertices"].dtype == np.float32 and r["normals"].dtype == np.float32
    assert np.all(np.abs(r["vertices"].astype(np.float64) - w) <= 0.5 * step * (1 + 1e-6) + 1e-6)
    assert np.all(np.abs(r["normals"] - m["normals"]) <= 0.5 / 127 + 1e-7)
