"""TEST INFRASTRUCTURE: a numpy stand-in for the ground-truth-map methods of `lidiff_b200._lib.Handle` (lb2_map_rehash /
lb2_map_scan), on top of the CPU fake of tests/fake_backend.py, so the host logic of lidiff_b200.maps and the map_from_scans CLI
can be exercised without a GPU.  `restate_scan` / `restate_map` restate the kernels' documented arithmetic in numpy fp32 (every
operation rounded, no FMA) and are also the yardstick of the GPU tests.  Tests install it by monkeypatching `_lib.get_handle`."""
import numpy as np
import torch

import fake_backend

AXIS_OFF = 1 << 20


def restate_scan(points, labels, pose12, voxel_size, div_mode):
    """(kept mask, transformed fp32 (n, 3), packed int64 voxel keys, in-range mask) of one scan"""
    p = np.asarray(points, dtype=np.float32).reshape(-1, 4)
    x, y, z, r = (p[:, j] for j in range(4))
    keep = np.sqrt(((x * x + y * y) + z * z) + r * r) > np.float32(3.5)
    if labels is not None:
        lab = np.asarray(labels).view(np.uint32) & np.uint32(0xFFFF)
        keep &= (lab > 1) & (lab < 252)
    m = np.asarray(pose12, dtype=np.float32).reshape(3, 4)
    w = np.stack([((m[k, 0] * x + m[k, 1] * y) + m[k, 2] * z) + m[k, 3] for k in range(3)], 1).astype(np.float32)
    vs = np.float32(voxel_size)
    q = w / vs if div_mode == 0 else w * (np.float32(1.0) / vs)
    f = np.floor(q)
    ok = np.all((f >= -AXIS_OFF) & (f < AXIS_OFF), axis=1)
    u = np.where(ok[:, None], f, 0).astype(np.int64) + AXIS_OFF
    keys = (u[:, 0] << 42) | (u[:, 1] << 21) | u[:, 2]
    return keep, w, keys, ok


def restate_map(scans, voxel_size, div_mode):
    """global first-occurrence de-duplication of the concatenated kept points: scans = [(points, labels, pose12)]"""
    ws, ks = [np.zeros((0, 3), np.float32)], [np.zeros(0, np.int64)]
    for points, labels, pose12 in scans:
        keep, w, keys, ok = restate_scan(points, labels, pose12, voxel_size, div_mode)
        if not ok[keep].all():
            raise ValueError("voxel index out of range")
        ws.append(w[keep])
        ks.append(keys[keep])
    w, k = np.concatenate(ws), np.concatenate(ks)
    _, first = np.unique(k, return_index=True)
    return w[np.sort(first)]


class FakeMapsHandle(fake_backend.FakeHandle):
    def __init__(self):
        super().__init__()
        self.tables = {}                 # keys tensor address -> {voxel key: map row}

    def new_map_table(self, cap):
        return (torch.empty(cap, dtype=torch.int64), torch.empty(2 * cap, dtype=torch.int32), cap)

    def map_rehash(self, old, table):
        self.launches += 1 if old is None else 2
        self.tables[table[0].data_ptr()] = dict(self.tables[old[0].data_ptr()]) if old is not None else {}

    def map_scan_scratch(self, n_cap):
        return torch.empty(16, dtype=torch.uint8)

    def map_scan(self, points, labels, pose12, voxel_size, div_mode, table, map_buf, map_n, out, scratch):
        n = points.shape[0]
        cap = table[2]
        assert cap >= 2 * (map_n + n) and map_buf.shape[0] >= map_n + n, "the caller must size the table and the map first"
        self.launches += 4
        known = self.tables[table[0].data_ptr()]
        keep, w, keys, ok = restate_scan(points.numpy(), None if labels is None else labels.numpy(), pose12, voxel_size, div_mode)
        out[1] = int(bool((keep & ~ok).any()))
        new = 0
        for i in np.nonzero(keep & ok)[0]:
            k = int(keys[i])
            if k not in known:
                known[k] = map_n + new
                map_buf[map_n + new] = torch.from_numpy(w[i])
                new += 1
        out[0] = new


def install(monkeypatch):
    """route the product's handle lookup to the CPU fake with the map stand-ins (host-logic tests only)"""
    from lidiff_b200 import _lib
    h = FakeMapsHandle()
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    return h
