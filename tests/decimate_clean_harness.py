"""TEST HARNESS of the decimation's topological-noise removal: ops.decimate(max_cut=, min_component=) driven over the
host-compiled bodies of csrc/decimate.cu (the library of tests/decimate_harness.py, which binds every perf_decimate_* entry
point), with numpy for the sorts and scans.  The CPU suite checks it against tests/decimate_clean_oracle.py, the GPU suite
the kernels against it."""
import numpy as np

from decimate_harness import NO_KEY, _exclusive, _ok, _p, adjacency, lib


def components(f, V):
    label = np.arange(V, dtype=np.int32)
    changed = np.zeros(1, np.int32)
    while True:
        changed[0] = 0
        _ok(lib().perf_decimate_components(_p(f), len(f), V, _p(label), _p(changed), None))
        if not changed[0]:
            return label


def drop_flags(pos, f, label, min_component):
    """-> (valive [V] uint8, falive [F] uint8, box [V,6] int32)."""
    V, F = len(pos), len(f)
    box = np.empty((V, 6), np.int32)
    box[:, :3], box[:, 3:] = 2 ** 31 - 1, -2 ** 31
    valive, falive = np.empty(V, np.uint8), np.empty(F, np.uint8)
    _ok(lib().perf_decimate_component_box(_p(pos), V, _p(f), F, _p(label), float(min_component), _p(box), _p(valive), _p(falive), None))
    return valive, falive, box


def compact(pos, quad, f, valive, falive):
    V2, F2 = int(valive.sum()), int(falive.sum())
    pos2, quad2, f2 = np.empty((V2, 3), np.float32), np.empty((V2, 10), np.float64), np.empty((F2, 3), np.int32)
    _ok(lib().perf_decimate_compact(_p(pos), _p(quad), len(pos), _p(valive), _p(_exclusive(valive)), _p(f), len(f), _p(falive),
                                    _p(_exclusive(falive)), _p(pos2), _p(quad2), _p(f2), None))
    return pos2, quad2, f2


def drop(pos, quad, f, min_component):
    label = components(f, len(pos))
    valive, falive, _ = drop_flags(pos, f, label, min_component)
    dropped = int(((label == np.arange(len(pos))) & (valive == 0)).sum())
    if dropped == 0:
        return pos, quad, f, 0
    return (*compact(pos, quad, f, valive, falive), dropped)


def cycles(pos, f, adj, off, max_cut):
    """-> (key [3F], third [3F], selected cycle half-edges ascending)."""
    V, F = len(pos), len(f)
    key, third = np.empty(3 * F, np.int64), np.full(3 * F, -1, np.int32)
    vmin = np.full(V, NO_KEY, np.int64)
    _ok(lib().perf_decimate_cycles(_p(pos), V, _p(f), F, _p(adj), _p(off), float(max_cut), _p(key), _p(third), _p(vmin), None))
    vmin2, sel = vmin.copy(), np.empty(3 * F, np.uint8)
    _ok(lib().perf_decimate_cycle_select(_p(f), F, V, _p(key), _p(third), _p(vmin), _p(vmin2), _p(sel), None))
    return key, third, np.nonzero(sel)[0].astype(np.int64)


def cut(pos, quad, f, adj, off, sel, third):
    V, F, n = len(pos), len(f), len(sel)
    pos2 = np.concatenate([pos, np.zeros((3 * n, 3), np.float32)])
    quad2 = np.concatenate([quad, np.zeros((3 * n, 10), np.float64)])
    f2 = np.concatenate([f, np.zeros((2 * n, 3), np.int32)])
    _ok(lib().perf_decimate_cut(_p(sel), n, _p(third), _p(pos2), _p(quad2), V, _p(f2), F, _p(adj), _p(off), None))
    return pos2, quad2, f2


def decimate(vertices, faces, target, max_cut=None, min_component=None, rounds=None, on_round=None):
    """ops.decimate with the new arguments on the host-compiled bodies -> (vertices [V',3] f32, faces [F',3] int32).
    ``rounds``, when a list, receives per round (kind, payload, faces after): ("collapse", sorted edge ids after the budget),
    ("cut", sorted cycle half-edge ids), ("drop", components dropped).  ``on_round(kind, vertices, faces)`` sees every mesh."""
    L = lib()
    pos = np.ascontiguousarray(vertices, np.float32).copy()
    f = np.ascontiguousarray(faces, np.int32).copy()
    V, F = len(pos), len(f)
    if F == 0:
        return pos, f

    def log(kind, payload):
        if rounds is not None:
            rounds.append((kind, payload, len(f)))
        if on_round is not None:
            on_round(kind, pos, f)
    adj, off = adjacency(f, V)
    flags = np.zeros(1, np.int32)
    _ok(L.perf_decimate_check(_p(f), F, V, _p(adj), _p(off), _p(flags), None))
    if flags[0]:
        raise ValueError(f"decimate: not a closed, consistently oriented, edge-manifold mesh (flags {int(flags[0])})")
    quad = np.empty((V, 10), np.float64)
    _ok(L.perf_decimate_quadrics(_p(pos), V, _p(f), F, _p(adj), _p(off), _p(quad), None))
    if min_component is not None:
        pos, quad, f, d = drop(pos, quad, f, min_component)
        V, F = len(pos), len(f)
        log("drop", d)
    while F > target:
        adj, off = adjacency(f, V)
        key = np.empty(3 * F, np.int64)
        place = np.empty((3 * F, 3), np.float32)
        vmin = np.full(V, NO_KEY, np.int64)
        _ok(L.perf_decimate_edges(_p(pos), _p(quad), V, _p(f), F, _p(adj), _p(off), _p(key), _p(place), _p(vmin), None))
        vmin2, sel = vmin.copy(), np.empty(3 * F, np.uint8)
        _ok(L.perf_decimate_select(_p(f), F, V, _p(key), _p(vmin), _p(vmin2), _p(sel), None))
        edges = np.nonzero(sel)[0].astype(np.int64)
        if len(edges) == 0:
            if max_cut is None:
                break
            _, third, cyc = cycles(pos, f, adj, off, max_cut)
            if len(cyc) == 0:
                log("cut", cyc)
                break
            pos, quad, f = cut(pos, quad, f, adj, off, cyc, third)
            log("cut", cyc)
            if min_component is not None:
                pos, quad, f, d = drop(pos, quad, f, min_component)
                log("drop", d)
            V, F = len(pos), len(f)
            continue
        need = (F - target + 1) // 2
        if len(edges) > need:
            edges = np.sort(edges[np.argsort(key[edges])[:need]])
        n = len(edges)
        valive, falive = np.ones(V, np.uint8), np.ones(F, np.uint8)
        _ok(L.perf_decimate_collapse(_p(edges), n, _p(pos), _p(quad), V, _p(f), F, _p(adj), _p(off), _p(place), _p(valive), _p(falive), None))
        pos, quad, f = compact(pos, quad, f, valive, falive)
        V, F = len(pos), len(f)
        log("collapse", edges)
    return pos, f
