"""TEST INFRASTRUCTURE: a CPU stand-in for `lidiff_b200._lib.Handle` so the HOST logic of the product
(operator surface wiring, engine orchestration, buffer/pointer plumbing, ctypes descriptors) can be
exercised without a GPU.  Every entry point is implemented with the oracle's primitives on CPU
memory reached through the same raw pointers the CUDA library would get.  Never shipped, never used
by the product: tests install it by monkeypatching `_lib.get_handle`."""
import ctypes as C

import numpy as np
import torch

from oracle import me_cpu as ome
from split_numerics import split


def _arr(ptr, shape, ctype, npdtype):
    n = int(np.prod(shape))
    if n == 0:
        return np.zeros(shape, npdtype)
    buf = (ctype * n).from_address(ptr)
    return np.frombuffer(buf, dtype=npdtype).reshape(shape)


def _f(ptr, shape):
    return _arr(ptr, shape, C.c_float, np.float32)


def _i(ptr, shape):
    return _arr(ptr, shape, C.c_int32, np.int32)


def _h(ptr, shape):
    return _arr(ptr, shape, C.c_uint16, np.float16)


def _read_act(f_ptr, h_ptr, rows, c):
    """an activation as float64: from the fp32 tensor, else from its fp16 split companion (row = [hi | lo])"""
    if f_ptr:
        return torch.from_numpy(_f(f_ptr, (rows, c)).copy()).double()
    hl = torch.from_numpy(_h(h_ptr, (rows, 2 * c)).astype(np.float32))
    return (hl[:, :c] + hl[:, c:]).double()


def _write_act(f_ptr, h_ptr, rows, c, y):
    y32 = y.float()
    if f_ptr:
        _f(f_ptr, (rows, c))[:] = y32.numpy()
    if h_ptr:
        _h(h_ptr, (rows, 2 * c))[:] = torch.cat(split(y32), 1).numpy()


class FakeHandle:
    def __init__(self):
        self.device = torch.device("cpu")
        self.grids = {}
        self.launches = 0
        self.status = 0
        self.emulate_tc = False

    # plumbing -------------------------------------------------------------------------------------
    def launch_count(self):
        return self.launches

    def read_status(self):
        s, self.status = self.status, 0
        return s

    def new_grid(self, n_cap):
        cap = 1 << max(4, (2 * n_cap - 1).bit_length())
        return (torch.empty(cap, dtype=torch.int64), torch.empty(2 * cap, dtype=torch.int32), cap)

    def unique_scratch(self, n_cap):
        return torch.empty(16, dtype=torch.uint8)

    def voxel_mean_scratch(self, m_cap, c):
        return torch.empty(16, dtype=torch.uint8)

    @staticmethod
    def _n(d_n, cap):
        return cap if d_n is None else min(int(d_n[0]), cap)

    # coords ---------------------------------------------------------------------------------------
    def quantize(self, x, resolution, div_mode, out):
        self.launches += 1
        out.copy_(ome.quantize(x, resolution, "div" if div_mode == 0 else "mul").reshape(out.shape))

    def unique_build(self, in_f, in_i, d_nin, n_cap, ts_floor, grid, out_coords, inverse, d_nout, scratch):
        self.launches += 6
        n = self._n(d_nin, n_cap)
        rows = torch.floor(in_f[:n]).long().numpy() if in_f is not None else in_i[:n].long().numpy()
        rows = rows.copy()
        if ts_floor > 0:
            rows[:, 1:] = np.floor_divide(rows[:, 1:], ts_floor) * ts_floor
        first, inv = ome.unique_first_occurrence(rows)
        M = first.shape[0]
        out_coords[:M] = torch.from_numpy(rows[first].astype(np.int32))
        if inverse is not None:
            inverse[:n] = torch.from_numpy(inv.astype(np.int32))
        d_nout[0] = M
        keys = ome.pack_keys(rows[first])
        order = np.argsort(keys, kind="stable")
        self.grids[grid[0].data_ptr()] = (keys[order], order)

    def voxel_mean(self, feats, inverse, n, c, d_m, m_cap, out, scratch):
        self.launches += 2
        M = self._n(d_m, m_cap)
        inv = inverse[:n].long()
        sums = torch.zeros(M, c)
        sums.index_add_(0, inv, feats[:n])
        cnt = torch.bincount(inv, minlength=M).float()
        out[:M] = sums / cnt[:, None]

    def kernel_map(self, grid_in, out_coords, d_nout, nout_cap, ks, step, nbr, nbr_stride, pair_count=None, row_mask=None):
        self.launches += 1
        n = self._n(d_nout, nout_cap)
        skeys, order = self.grids[grid_in[0].data_ptr()]
        Cq = out_coords[:n].long().numpy()
        r = np.arange(ks)
        kz, ky, kx = np.meshgrid(r, r, r, indexing="ij")
        offs = np.stack([kx.reshape(-1), ky.reshape(-1), kz.reshape(-1)], 1)
        if ks % 2 == 1:
            offs = offs - ks // 2
        nb = nbr.reshape(-1)[: ks ** 3 * nbr_stride].view(ks ** 3, nbr_stride)
        for k, off in enumerate(offs * step):
            q = Cq.copy()
            q[:, 1:] += off[None, :]
            ok = (np.abs(q[:, 1:]) < ome.AXIS_OFF).all(1)
            qk = ome.pack_keys(np.where(ok[:, None], q, 0))
            pos = np.minimum(np.searchsorted(skeys, qk), max(skeys.shape[0] - 1, 0))
            hit = ok & (skeys[pos] == qk) if skeys.shape[0] else np.zeros(n, bool)
            res = np.where(hit, order[pos], -1).astype(np.int32)
            nb[k, :n] = torch.from_numpy(res)
            nb[k, n:nout_cap] = -1
            if pair_count is not None:
                pair_count += int(hit.sum())
            if row_mask is not None:
                if k == 0:
                    row_mask[:nout_cap] = 0
                row_mask[:n] |= torch.from_numpy((hit.astype(np.int64) << k).astype(np.int32))

    def kernel_map_self(self, grid, coords, d_n, n_cap, step, nbr, nbr_stride, pair_count=None, row_mask=None):
        self.kernel_map(grid, coords, d_n, n_cap, 3, step, nbr, nbr_stride, pair_count, row_mask)

    def row_order_scratch_bytes(self, n_cap):
        return 1024

    def row_order(self, row_mask, d_n, n_cap, kvol, perm, scratch, coords=None, coord_shift=0):
        self.launches += 3 if kvol <= 8 else 6
        n = self._n(d_n, n_cap)
        m = row_mask[:n].long() & 0xFFFFFFFF
        if kvol <= 8:
            b = m & 0xFF
        else:                                        # [>= 2 off-centre neighbours | mask without the centre bit]
            extras = m & ~(1 << 13)
            pop = sum(((extras >> j) & 1) for j in range(27))
            b = ((pop >= 2).long() << 26) | ((m >> 14) << 13) | (m & 0x1FFF)
        order = torch.argsort(b, stable=True)
        perm[:n] = torch.flip(order, [0]).int() if n > 3 else order.int()     # any in-bucket order is legal; scramble a bit
        perm[:n] = order.int()

    def tile_order(self, row_mask, row_perm, d_n, n_cap, order128, order256, scratch):
        self.launches += 2
        n = self._n(d_n, n_cap)
        m = (row_mask[:n][row_perm[:n].long()] if row_perm is not None else row_mask[:n]).long() & 0xFFFFFFFF
        for T, out in ((128, order128), (256, order256)):
            nt = (n + T - 1) // T
            cost = torch.tensor([bin(int(torch.tensor(0) if m[t * T:(t + 1) * T].numel() == 0 else
                                         torch.from_numpy(np.bitwise_or.reduce(m[t * T:(t + 1) * T].numpy(), keepdims=True))[0])).count("1") for t in range(nt)])
            out[:] = -1
            out[:nt] = torch.argsort(-cost, stable=True).int()

    # conv -----------------------------------------------------------------------------------------
    def packed_weight_bytes(self, kvol, cin, cout):
        return 0

    def pack_weights(self, w):
        # the fake keeps the fp32 weight itself as the "packed" image so the scatter path can be exercised
        return w.detach().clone() if self.emulate_tc else None

    def scatter_supported(self, c1, c2, cout, kvol):
        return self.emulate_tc and (c1 + c2) % 16 == 0 and cout % 32 == 0 and cout <= 128

    def pair_list(self, nbr, nbr_stride, d_nout, nout_cap, kvol, skip_k, pair_in, pair_out, koff, tile_off, scratch):
        self.launches += 3
        n = self._n(d_nout, nout_cap)
        nb = nbr.reshape(-1)[: kvol * nbr_stride].view(kvol, nbr_stride)[:, :n]
        a = t = 0
        for k in range(kvol):
            koff[k], tile_off[k] = a, t
            if k == skip_k:
                continue
            o = torch.nonzero(nb[k] >= 0)[:, 0]
            o = o[torch.randperm(o.shape[0])]                       # order inside an offset is unspecified
            pair_in[a:a + o.shape[0]] = nb[k][o]
            pair_out[a:a + o.shape[0]] = o.int()
            a += o.shape[0]
            t += (o.shape[0] + 127) // 128
        koff[kvol], tile_off[kvol] = a, t

    def spconv_scatter(self, d):
        self.launches += 2
        koff = _i(d.koff, (d.kvol + 1,))
        P = int(koff[d.kvol])
        pin, pout = _i(d.pair_in, (P,)).astype(np.int64), _i(d.pair_out, (P,)).astype(np.int64)
        ctot = d.c1 + d.c2
        W = torch.from_numpy(_f(d.weight_packed, (d.kvol, ctot, d.cout)).copy()).double()
        M = min(int(_i(d.d_zero_rows, (1,))[0]), d.zero_rows_cap) if d.d_zero_rows else d.zero_rows_cap
        rows_in = int(pin.max()) + 1 if P else 0
        for p in range(d.npass):
            out = _f(d.out[p], (M, d.cout))
            if d.zero_rows_cap > 0:
                out[:] = 0
            x = torch.from_numpy(_f(d.in1[p], (rows_in, d.c1)).copy())
            if d.c2:
                x = torch.cat([x, torch.from_numpy(_f(d.in2[p], (rows_in, d.c2)).copy())], 1)
            x = x.double()
            acc = torch.from_numpy(out.copy()).double()
            for k in range(d.kvol):
                a, b = int(koff[k]), int(koff[k + 1])
                if b > a:
                    acc.index_add_(0, torch.from_numpy(pout[a:b]), x[torch.from_numpy(pin[a:b])] @ W[k])
            out[:] = acc.float().numpy()

    def spconv(self, d, algo=0):
        self.launches += 1
        M = d.mout_cap if not d.d_mout else min(int(_i(d.d_mout, (1,))[0]), d.mout_cap)
        if d.row_perm:          # scheduling hint only: must be a permutation of the M rows
            assert np.array_equal(np.sort(_i(d.row_perm, (M,))), np.arange(M)), "row_perm is not a permutation"
        ctot = d.c1 + d.c2
        W = torch.from_numpy(_f(d.weight, (d.kvol, ctot, d.cout)).copy()).double()
        nbr = _i(d.nbr, (d.kvol, d.nbr_stride))[:, :M] if d.nbr else np.arange(M, dtype=np.int32)[None]
        if d.row_mask and d.nbr:  # hint only: must agree with the map it describes
            want = np.zeros(M, np.int64)
            for k in range(d.kvol):
                want |= (nbr[k] >= 0).astype(np.int64) << k
            assert np.array_equal(_i(d.row_mask, (M,)).astype(np.int64) & 0xFFFFFFFF, want), "row_mask disagrees with nbr"
        rows_in = int(nbr.max()) + 1 if nbr.size else 0
        for p in range(d.npass):
            io = d.io[p]
            x = _read_act(io.in1, io.in1_h, rows_in, d.c1)
            if d.c2:
                x = torch.cat([x, _read_act(io.in2, io.in2_h, rows_in, d.c2)], 1)
            y = torch.zeros(M, d.cout, dtype=torch.float64)
            for k in range(d.kvol):
                o = np.nonzero(nbr[k] >= 0)[0]
                if o.size:
                    y[torch.from_numpy(o)] += x[torch.from_numpy(nbr[k][o].astype(np.int64))] @ W[k]
            if io.pre_add:
                y = y + torch.from_numpy(_f(io.pre_add, (M, d.cout)).copy()).double()
            if d.scale:
                y = y * torch.from_numpy(_f(d.scale, (d.cout,)).copy()).double() + torch.from_numpy(_f(d.shift, (d.cout,)).copy()).double()
            if io.residual or io.residual_h:
                y = y + _read_act(io.residual, io.residual_h, M, d.cout)
            if d.relu:
                y = torch.relu(y)
            _write_act(io.out, io.out_h, M, d.cout, y)
            if io.out_gated or io.out_gated_h:
                g = y
                if io.gate_table:
                    gi = _i(io.gate_idx, (M,)).astype(np.int64) if io.gate_idx else np.zeros(M, np.int64)
                    rows_g = int(gi.max()) + 1 if M else 0
                    tab = torch.from_numpy(_f(io.gate_table, (rows_g, d.cout)).copy()).double()
                    g = y * tab[torch.from_numpy(gi)]
                _write_act(io.out_gated, io.out_gated_h, M, d.cout, g)

    # misc -----------------------------------------------------------------------------------------
    def nn_match(self, q, d_nq, nq_cap, k, d_nk, nk_cap, batch_scale, idx):
        self.launches += 1
        nq, nk = self._n(d_nq, nq_cap), self._n(d_nk, nk_cap)
        qq, kk = q[:nq].double(), k[:nk].double()
        if batch_scale == 0:
            qq, kk = qq.clone(), kk.clone()
            qq[:, 0] *= 1e9
            kk[:, 0] *= 1e9
        out = torch.empty(nq, dtype=torch.int64)
        for s in range(0, nq, 4096):
            d = ((qq[s:s + 4096, None, :] - kk[None]) ** 2).sum(-1)
            out[s:s + 4096] = torch.argmin(d, 1)
        idx[:nq] = out.int()

    def nn_match_grid(self, q, d_nq, nq_cap, k, d_nk, nk_cap, key_grid, key_stride, max_ring, idx):
        self.nn_match(q, d_nq, nq_cap, k, d_nk, nk_cap, 0, idx)

    def nn_tree(self, k, d_nk, nk_cap, out=None):
        self.launches += 12
        return (k, d_nk)

    def nn_match_tree(self, q, d_nq, nq_cap, tree, nk_cap, idx, k=None, hint_of=None, hint_idx=None):
        self.nn_match(q, d_nq, nq_cap, tree[0], tree[1], nk_cap, 0, idx)

    def nn_table(self, k, d_nk, nk_cap):
        return torch.zeros(16, dtype=torch.uint8)

    def nn_match_table(self, q, d_nq, nq_cap, k, d_nk, nk_cap, table, key_stride, max_ring, idx):
        self.nn_match(q, d_nq, nq_cap, k, d_nk, nk_cap, 0, idx)

    @staticmethod
    def _act(v, act):
        return torch.nn.functional.leaky_relu(v, 0.1) if act == 1 else (torch.tanh(v) if act == 2 else v)

    def linear(self, x, ldx, w, b, addend, ld_add, m_cap, d_m, n_in, n_out, act, y, ldy, prebias=None, pre_act=0):
        self.launches += 1
        M = self._n(d_m, m_cap)
        xs = torch.as_strided(x, (M, n_in), (ldx, 1))
        if prebias is not None:
            xs = self._act(xs + prebias, pre_act)
        v = xs.double() @ w.double().t()
        if b is not None:
            v = v + b.double()
        if addend is not None:
            v = v + torch.as_strided(addend, (M, n_out), (ld_add, 1)).double()
        torch.as_strided(y, (M, n_out), (ldy, 1)).copy_(self._act(v, act).float())

    def gate_mul(self, x, table, idx, d_m, m_cap, c, out, out_h=None):
        self.launches += 1
        M = self._n(d_m, m_cap)
        g = table[idx[:M].long()] if idx is not None else table[0:1]
        y = x[:M] * g
        if out is not None:
            out[:M] = y
        if out_h is not None:
            out_h[:M] = torch.cat(split(y), 1)

    def head_mlp(self, x, ldx, x_pass_stride, w0, b0, w1, b1, m_cap, d_m, n_in, n_hid, n_out, out_act, npass, y, ldy, y_pass_stride):
        self.launches += 1
        M = self._n(d_m, m_cap)
        for p in range(npass):
            xs = torch.as_strided(x, (M, n_in), (ldx, 1), x.storage_offset() + p * x_pass_stride).double()
            hid = torch.nn.functional.leaky_relu(xs @ w0.double().t() + (b0.double() if b0 is not None else 0), 0.1)
            v = hid @ w1.double().t() + (b1.double() if b1 is not None else 0)
            torch.as_strided(y, (M, n_out), (ldy, 1), y.storage_offset() + p * y_pass_stride).copy_(self._act(v, out_act).float())

    def gather_rows(self, src, idx, n, c, out):
        self.launches += 1
        out[:n] = src[idx[:n].long()]

    def guidance_dpm_step(self, eps_c, eps_u, inverse, x_t, x_init, noise, x0_state, n_points, cf, eps_out, x_next, coord_next, batch_col=None):
        self.launches += 1
        n = n_points
        inv = inverse[:n].long() if inverse is not None else torch.arange(n)
        ec, eu = eps_c[inv], eps_u[inv]
        eps = eu + torch.tensor(cf.guidance_w, dtype=torch.float32) * (ec - eu)
        if eps_out is not None:
            eps_out[:n] = eps
        f32 = lambda v: torch.tensor(v, dtype=torch.float32)
        sample = x_t[:n] - x_init[:n]
        x0 = (sample - f32(cf.sigma_s) * eps) / f32(cf.alpha_s)
        prev = f32(cf.c_sample) * sample + f32(cf.c_x0) * x0
        if cf.second_order:
            prev = prev + 0.5 * f32(cf.c_x0) * (f32(cf.inv_r0) * (x0 - x0_state[:n]))
        prev = prev + f32(cf.c_noise) * noise[:n].float()       # fp32 product (diffusers: fp32 noise), then promoted
        x0_state[:n] = x0
        xn = (x_init[:n] + prev).float()
        x_next[:n] = xn
        if coord_next is not None:
            coord_next[:n, 1:] = ome.quantize(xn, cf.resolution, "div" if cf.div_mode == 0 else "mul")
            coord_next[:n, 0] = 0 if batch_col is None else batch_col[:n]

    def farthest_point_sample(self, pts, n, n_samples, out_idx, dist):
        from oracle.pipeline import farthest_point_sample
        self.launches += 1
        p = pts[:n].numpy()
        sel = np.empty(n_samples, np.int64)
        d = np.full(n, np.inf)
        cur = 0
        for i in range(n_samples):
            sel[i] = cur
            d = np.minimum(d, ((p - p[cur]) ** 2).sum(1))
            cur = int(np.argmax(d))
        out_idx[:n_samples] = torch.from_numpy(sel.astype(np.int32))


def install(monkeypatch, emulate_tc=False):
    """route the product's handle lookup to the CPU fake (host-logic tests only)"""
    from lidiff_b200 import _lib, me
    h = FakeHandle()
    h.emulate_tc = emulate_tc
    monkeypatch.setattr(_lib, "get_handle", lambda device=None: h)
    monkeypatch.setattr(me, "_require_cuda", lambda t, what: None)
    return h
