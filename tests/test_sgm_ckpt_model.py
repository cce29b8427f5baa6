"""CPU: the bookkeeping of the fused pipeline's sgm2 schedule (csrc/sgm.cu, adc_sgm2_ckpt) restated in numpy, against
oracle.sgm2 of a zero accumulator, bit for bit.  The forward scans (rightward, downward) keep only the line state
entering every CK-th step; the backward scans (leftward, upward) recompute the forward values block by block from
those states, last block first, and accumulate ((0 + right) + left) + down) + up.  Shapes sit below, on, one above and
off the checkpoint spacing, so a block-edge mistake (an off-by-one checkpoint, a block restarted as a line start, a
partial last block) shows here before it is looked for on the GPU."""
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("dispatch_cases", os.path.join(ROOT, "tests", "dispatch_cases.py"))
dc = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(dc)

CK_H, CK_V = 16, 8          # sgm.cu SGM_CK_H / SGM_CK_V
f32 = np.float32


class Scans:
    """one step of each scan direction for all its lines at once, expression for expression as adcensus.cu:567-617"""

    def __init__(self, x0, x1, vol, params, direction):
        self.x0, self.x1, self.vol, self.direction = x0, x1, vol, direction
        pi1, pi2, tau, alpha1, q1, q2 = (f32(v) for v in params)
        self.tau, self.alpha1 = tau, alpha1
        self.pen = ((pi1, pi2), (pi1 / (q1 * q2), pi2 / (q1 * q2)), (pi1 / q1, pi2 / q1))
        self.H, self.W, self.D = vol.shape

    def pixel(self, sd, s):
        """(ys, xs) of step s on every line, and the scan's (dy, dx)"""
        H, W = self.H, self.W
        if sd < 2:
            x = s if sd == 0 else W - 1 - s
            return np.arange(H), np.full(H, x), 0, (1 if sd == 0 else -1)
        y = s if sd == 2 else H - 1 - s
        return np.full(W, y), np.arange(W), (1 if sd == 2 else -1), 0

    def step(self, sd, s, prev):
        """values of step s from the line state `prev` ((lines, D)); None: the first pixel of the line"""
        ys, xs, dy, dx = self.pixel(sd, s)
        cin = self.vol[ys, xs]
        if prev is None:
            return cin.copy()
        D, W = self.D, self.W
        m = prev.copy()
        for i in (256, 128, 64, 32, 16, 8, 4, 2, 1):                                       # :579-584
            n = min(i, D - i)
            if n > 0:
                m[:, :n] = np.where(m[:, i:i + n] < m[:, :n], m[:, i:i + n], m[:, :n])
        m = m[:, :1]
        d1 = np.abs(self.x0[ys, xs] - self.x0[ys - dy, xs - dx])[:, None]                  # :587
        xx = xs[:, None] + np.arange(D)[None, :] * self.direction
        inside = (xx >= 0) & (xx < W) & (xx - dx >= 0) & (xx - dx < W)
        xc = np.clip(xx, 0, W - 1)
        d2 = np.where(inside, np.abs(self.x1[ys[:, None], xc] - self.x1[ys[:, None] - dy, np.clip(xc - dx, 0, W - 1)]), f32(10))
        lo, hi = (d1 < self.tau) & (d2 < self.tau), (d1 > self.tau) & (d2 > self.tau)      # :596-605
        P1 = np.where(lo, self.pen[0][0], np.where(hi, self.pen[1][0], self.pen[2][0])).astype(f32)
        P2 = np.where(lo, self.pen[0][1], np.where(hi, self.pen[1][1], self.pen[2][1])).astype(f32)
        cost = np.fmin(prev, m + P2)                                                       # :607
        Pm = P1 / self.alpha1 if sd == 2 else P1
        Pp = P1 / self.alpha1 if sd == 3 else P1
        cost[:, 1:] = np.fmin(cost[:, 1:], prev[:, :-1] + Pm[:, 1:])                       # :609
        cost[:, :-1] = np.fmin(cost[:, :-1], prev[:, 1:] + Pp[:, :-1])                     # :612
        return (cin + cost) - m                                                            # :615

    def forward(self, sd, ck):
        """sgm_fwd_kernel: checkpoint b = the state entering step b * ck, b >= 1"""
        L = self.W if sd == 0 else self.H
        prev, cks = None, {}
        for s in range(L):
            prev = self.step(sd, s, prev)
            if (s + 1) % ck == 0 and s + 1 < L:
                cks[(s + 1) // ck] = prev
        assert sorted(cks) == list(range(1, -(-L // ck)))
        return cks

    def block(self, sd, cks, b, ck):
        """the forward values of the steps of block b, recomputed from its checkpoint"""
        L = self.W if sd == 0 else self.H
        prev, vals = cks.get(b), []
        assert (prev is None) == (b == 0)
        for s in range(b * ck, min(L, (b + 1) * ck)):
            prev = self.step(sd, s, prev)
            vals.append(prev)
        return vals


def ckpt_schedule(x0, x1, vol, params, direction):
    sc = Scans(x0, x1, vol, params, direction)
    H, W, _ = vol.shape
    out = np.empty_like(vol)
    ckh, ckv = sc.forward(0, CK_H), sc.forward(2, CK_V)
    # sgm_bwd_h_kernel: the leftward scan, the rightward values of a block recomputed before it reaches the block
    left, r = None, None
    for s in range(W):
        x = W - 1 - s
        if s == 0 or (x + 1) % CK_H == 0:
            b = x // CK_H
            r, x0b = sc.block(0, ckh, b, CK_H), b * CK_H
        left = sc.step(1, s, left)
        out[:, x] = (f32(0) + r[x - x0b]) + left
    # sgm_bwd_v_kernel: per block of rows from the bottom, the downward values recomputed, then the upward scan over them
    up = None
    for b in range(-(-H // CK_V) - 1, -1, -1):
        dn, y0 = sc.block(2, ckv, b, CK_V), b * CK_V
        for y in range(min(H, y0 + CK_V) - 1, y0 - 1, -1):
            up = sc.step(3, H - 1 - y, up)
            out[y] = (out[y] + dn[y - y0]) + up
    return out


SHAPES = [(1, 2, 3), (1, 16, 5), (7, 15, 4), (8, 16, 6), (9, 17, 5), (17, 33, 9), (24, 48, 3), (25, 37, 7)]


@pytest.mark.parametrize("direction", [-1, 1])
@pytest.mark.parametrize("H,W,D", SHAPES, ids=["H%dW%dD%d" % s for s in SHAPES])
def test_ckpt_bookkeeping_matches_oracle(oracle, H, W, D, direction):
    for params in (dc.SGM_TIE, dc.SGM_TEN):
        c = dc.SGMCase(H, W, D, 0, 0, params, dc.sgm_k(D), False)
        x0, x1, vol = dc.sgm_inputs(c, direction)
        want = oracle.sgm2(x0, x1, vol, *params, direction)
        got = ckpt_schedule(x0, x1, vol, params, direction)
        assert np.array_equal(got, want, equal_nan=True), (params, np.argwhere(~((got == want) | np.isnan(got) & np.isnan(want)))[:5])
        z = want == 0
        assert np.array_equal(np.signbit(got[z]), np.signbit(want[z]))
