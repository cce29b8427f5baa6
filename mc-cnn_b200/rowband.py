"""One stereo pair split by ROW BANDS over N GPUs (BASELINE.json config 5: a Middlebury-scale
volume), one process per GPU, torch.distributed (NCCL over NVLink) for the exchanges.

Which stages need an exchange follows from the reference's data dependences, not
from BASELINE.json's wording:

* StereoJoin, fix_border, the permutes, argmin, sub-pixel: row-local -> no communication;
* cross: needs image rows +- L1 -> both (small) images are replicated on every rank;
* cbca: the vertical arm reaches halo = max(L1,2)-1 rows into the neighbouring bands PER ITERATION.  A block of n
  iterations is run on the band extended by n * halo rows on either side (the valid part shrinks by `halo` rows per
  iteration and ends on the band): for the first block (cbca_i1) the extension costs nothing but arithmetic -- the
  features are replicated, StereoJoin simply covers the extended rows -- and the second block (cbca_i2, after SGM)
  needs ONE halo exchange with the two neighbours instead of one per iteration (falls back to one exchange per
  iteration when n * halo rows exceed a neighbour's band);
* sgm2: the two horizontal passes are band-local.  The two vertical passes are serial chains over the rows: they run as a
  WAVEFRONT over column chunks -- rank r scans its rows of chunk k as soon as rank r-1 (down pass; r+1 for the up pass)
  has sent the line state of its last row for that chunk (W/K x D floats), and passes its own last row's state on.
  Only that boundary state crosses a band, not the volumes; the pipeline fill costs (N-1)/K of
  a pass.  Direction order and therefore the accumulation order (right, left, down, up) are the reference's =>
  results are bit-identical to the single-GPU pipeline in its exact mode (tests/test_rowband_*.py);
* LR check / interpolations / median / bilateral work on H x W maps: the disparity maps are
  all-gathered (tiny) and these stages run replicated; sub-pixel refinement reads the band's own
  left volume.

The operators are injected (``ops``), so the same driver runs on the CUDA library (CudaOps) and,
in the CPU tests, on any object with the same methods over CPU tensors.
"""
import math

import torch
import torch.distributed as dist


def split(n, parts, i):
    """[lo, hi) of part i when n items are cut into `parts` nearly equal contiguous pieces"""
    return (n * i) // parts, (n * (i + 1)) // parts


class Comm:
    """Thin layer over torch.distributed point-to-point ops (works with nccl and gloo)."""

    def __init__(self):
        self.on = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        self.rank = dist.get_rank() if self.on else 0
        self.world = dist.get_world_size() if self.on else 1

    def exchange(self, sends, recvs):
        """sends: {peer: tensor}, recvs: {peer: empty tensor to fill}; all in flight together."""
        if not self.on:
            return
        ops = [dist.P2POp(dist.isend, t.contiguous(), p) for p, t in sends.items() if p != self.rank]
        ops += [dist.P2POp(dist.irecv, t, p) for p, t in recvs.items() if p != self.rank]
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()

    def all_gather_rows(self, band, H):
        """band: this rank's rows (Hb, W) of an H x W map -> the full map on every rank"""
        if not self.on:
            return band
        W = band.shape[-1]
        full = band.new_empty((H, W))
        y0, y1 = split(H, self.world, self.rank)
        full[y0:y1] = band
        sends = {p: band for p in range(self.world)}
        recvs = {}
        for p in range(self.world):
            a, b = split(H, self.world, p)
            recvs[p] = full[a:b]
        self.exchange(sends, recvs)
        return full

    def send(self, t, peer):
        """stream-ordered (nccl) / blocking (gloo) point-to-point send of a contiguous tensor"""
        if self.on:
            dist.send(t, peer)

    def recv(self, t, peer):
        if self.on:
            dist.recv(t, peer)

    def halo(self, vol, n):
        """vol (D, Hb, W): returns (rows from the band above, rows from the band below), each
        (D, <=n, W), empty at the image border"""
        D, Hb, W = vol.shape
        top = vol.new_empty((D, n if self.rank > 0 else 0, W))
        bot = vol.new_empty((D, n if self.rank < self.world - 1 else 0, W))
        if not self.on or n == 0:
            return vol.new_empty((D, 0, W)), vol.new_empty((D, 0, W))
        sends, recvs = {}, {}
        if self.rank > 0:
            sends[self.rank - 1] = vol[:, :n, :]
            recvs[self.rank - 1] = top
        if self.rank < self.world - 1:
            sends[self.rank + 1] = vol[:, Hb - n:, :]
            recvs[self.rank + 1] = bot
        # the two neighbours are distinct peers, so one batch carries both directions
        self.exchange(sends, recvs)
        return top, bot


def stereo_predict_rowband(ops, featL, featR, imgL, imgR, D, opt, comm=None, chunks=None):
    """main.lua:929-1082 (arch 'fast') with the rows of one pair split over the ranks of `comm`.

    featL/featR (C,H,W) and imgL/imgR (H,W) are the FULL tensors on every rank (only this rank's
    rows of the features are read).  `chunks`: column chunks of the vertical SGM wavefront (default: 4 per rank, at
    least 32 columns each).  Returns the full (H,W) disparity map on every rank.  Only the full chain: parameters with
    ``sm_terminate`` / ``sm_skip`` set are refused before any work (run them on one GPU through the fused pipeline).
    """
    for k in ("sm_terminate", "sm_skip"):
        if getattr(opt, k, 0):
            raise ValueError("row-band stereo_predict runs the full chain only: -%s is not supported (use the "
                             "single-GPU pipeline)" % k)
    comm = comm or Comm()
    H, W = imgL.shape
    N, r = comm.world, comm.rank
    y0, y1 = split(H, N, r)
    Hb = y1 - y0
    max_arm = max(int(opt.L1), 2)
    halo = max_arm - 1 if (opt.cbca_i1 + opt.cbca_i2) > 0 else 0
    band_min = min(split(H, N, p)[1] - split(H, N, p)[0] for p in range(N))
    if N > 1:
        assert band_min >= max(halo, 1), "bands thinner than the CBCA halo"
        assert max_arm <= 14, "row-band CBCA supports arms up to 14 pixels"
    # column chunks of the vertical wavefront: a chunk's scan is latency-bound (Hb serial steps) unless it is wide, and the chain
    # costs (N - 1 + K) chunk times: K = N is the measured sweet spot (K = 4 N made 39 hops of 94 columns at Middlebury size)
    K = chunks if chunks else max(1, min(N, W // 32)) if N > 1 else 1

    # first CBCA block on the band extended by cbca_i1 * halo rows: StereoJoin covers the extension (features are replicated)
    e1 = halo * int(opt.cbca_i1)
    ya, yb = max(0, y0 - e1), min(H, y1 + e1)
    volL, volR = ops.stereo_join(featL[:, ya:yb].contiguous(), featR[:, ya:yb].contiguous(), D)     # :946-947
    ops.fix_border(volL, opt.border, -1)                                                             # :948
    ops.fix_border(volR, opt.border, 1)                                                              # :949
    x0c = ops.cross(imgL, opt.L1, opt.tau1)                                                          # :995 (full image)
    x1c = ops.cross(imgR, opt.L1, opt.tau1)                                                          # :996

    def band_arms(arms, a, b):
        """arms of rows [a, b) in the coordinates of that sub-image; vertical end-points clamped to it
        (only rows whose outputs are discarded are affected)"""
        q = arms[:, a:b].clone()
        q[2] = torch.clamp(q[2] - a, min=-1)
        q[3] = torch.clamp(q[3] - a, max=b - a)
        return q.contiguous()

    def cbca_block(ext, a, b, n, direction):
        """n iterations on the extended band rows [a, b) (which hold valid data for all of [a, b)); rows closer than
        n * halo to an artificial edge end up invalid and are cut off by the caller"""
        if n == 0:
            return ext
        a0, a1 = band_arms(x0c, a, b), band_arms(x1c, a, b)
        for _ in range(n):
            ext = ops.cbca(a0, a1, ext, direction, max_arm)
        return ext

    def cbca_exchanging(vol, n, direction):
        """n iterations on the band [y0, y1): one exchange of n * halo rows when the neighbours hold that many, else one
        exchange of `halo` rows per iteration"""
        if n == 0 or halo == 0 or N == 1:
            return cbca_block(vol, y0, y1, n, direction)
        steps = [n] if n * halo <= band_min else [1] * n
        for m in steps:
            top, bot = comm.halo(vol, m * halo)
            ext = torch.cat([top, vol, bot], dim=1).contiguous() if (top.shape[1] or bot.shape[1]) else vol
            out = cbca_block(ext, y0 - top.shape[1], y1 + bot.shape[1], m, direction)
            vol = out[:, top.shape[1]: top.shape[1] + Hb].contiguous()
        return vol

    def vertical_wavefront(tab, cost, acc, direction, sd):
        """one vertical pass (sd 2 down, 3 up) chained over the ranks, column chunk by column chunk"""
        prev, nxt = (r + 1, r - 1) if sd == 3 else (r - 1, r + 1)      # in scan order
        has_prev, has_next = 0 <= prev < N, 0 <= nxt < N
        st_in = ops.new_state(W, D, cost) if has_prev else None
        st_out = ops.new_state(W, D, cost) if has_next else None
        for k in range(K):
            xa, xb = split(W, K, k)
            if xa == xb:
                continue
            if has_prev:
                comm.recv(st_in[xa:xb], prev)
            ops.sgm_rows(tab, cost, acc, H, y0, opt, direction, 1 << sd, False, xa, xb, st_in, st_out)
            if has_next:
                comm.send(st_out[xa:xb], nxt)

    disp = {}
    vol_left = None
    # main.lua:954-955: without the LR check (mb) only direction -1 is consumed
    for direction in ((1, -1) if opt.lr_check else (-1,)):                                           # :955
        ext = volL if direction == -1 else volR                                                      # :986
        ext = cbca_block(ext, ya, yb, int(opt.cbca_i1), direction)                                   # :998-1001
        vol = ext[:, y0 - ya: y0 - ya + Hb].contiguous() if (ya != y0 or yb != y1) else ext
        for _ in range(opt.sgm_i):                                                                   # :1008-1020
            tab = ops.sgm_tables(imgL, imgR, D, opt, direction)
            cost = ops.to_hwd(vol)                                                                   # (Hb, W, D)
            acc = getattr(ops, "new_acc", ops.zeros_like)(cost)                                      # :1014 (zero by contract, see new_acc)
            ops.sgm_rows(tab, cost, acc, H, y0, opt, direction, 3, True, 0, W, None, None)           # right, left: band-local
            vertical_wavefront(tab, cost, acc, direction, 2)                                         # down
            vertical_wavefront(tab, cost, acc, direction, 3)                                         # up
            vol = ops.from_hwd_div4(acc)                                                             # :1017-1020
        vol = cbca_exchanging(vol, int(opt.cbca_i2), direction)                                      # :1035-1038
        disp[direction] = comm.all_gather_rows(ops.argmin(vol), H)                                   # :1049-1050
        if direction == -1:
            vol_left = vol

    d = disp[-1]
    if opt.lr_check:                                                                                 # :1054-1066
        outlier = ops.outlier_detection(disp[-1], disp[1], D)
        d = ops.interpolate_occlusion(d, outlier)
        d = ops.interpolate_mismatch(d, outlier)
    sub = ops.subpixel(d[y0:y1].contiguous(), vol_left, D)                                           # :1068 (band-local)
    d = comm.all_gather_rows(sub, H)

    def band_filter(fn, full, r):
        """an H x W filter of radius r rows computed for this rank's rows only (on the band extended by r rows of the gathered
        map: the slice's edges are image edges exactly where the image ends), then gathered again"""
        a, b = max(0, y0 - r), min(H, y1 + r)
        o = fn(full[a:b].contiguous())
        return comm.all_gather_rows(o[y0 - a: y0 - a + Hb].contiguous(), H)

    d = band_filter(lambda t: ops.median2d(t, 5), d, 2)                                              # :1073
    kr = int(math.ceil(float(opt.blur_sigma) * 3))                                                   # main.lua:529: kernel radius
    return band_filter(lambda t: ops.mean2d(t, opt.blur_sigma, opt.blur_t), d, kr)                   # :1078


class CudaOps:
    """The operators on the CUDA library (torch CUDA tensors in, out)."""

    def __init__(self, device):
        self.device = device

    def stereo_join(self, fL, fR, D):
        from . import adcensus

        C, Hb, W = fL.shape
        vols = torch.empty((2, D, Hb, W), device=fL.device, dtype=torch.float32)
        adcensus.fill_nan(vols)
        adcensus.StereoJoin(fL[None], fR[None], vols[0:1], vols[1:2])
        return vols[0], vols[1]

    def fix_border(self, vol, n, direction):
        from . import adcensus

        adcensus.fix_border(vol[None], n, direction)

    def cross(self, img, L1, tau1):
        from . import adcensus

        out = torch.empty((1, 4) + tuple(img.shape), device=img.device, dtype=torch.float32)
        adcensus.cross(img[None].contiguous(), out, L1, tau1)
        return out[0]

    def cbca(self, x0c, x1c, vol, direction, max_arm):
        from . import adcensus

        out = torch.empty_like(vol)
        adcensus.cbca(x0c[None], x1c[None], vol[None], out[None], direction, max_arm=max_arm)
        return out

    def to_hwd(self, vol):
        from . import adcensus

        return adcensus.transpose_dhw_to_hwd(vol[None])[0]

    def from_hwd_div4(self, acc):
        from . import adcensus

        return adcensus.transpose_hwd_to_dhw_div4(acc[None])[0]

    def zeros_like(self, t):
        return torch.zeros_like(t)

    def new_acc(self, t):
        """the SGM accumulator of main.lua:1014: the first launch on it is the horizontal pair with zero_out = True, which never
        reads it and writes every element -- no memset needed on this backend"""
        return torch.empty_like(t)

    def sgm_band(self, imgL, imgR, cost, acc, Ht, Wt, yoff, xoff, opt, direction, pass_mask, zero_out):
        from . import adcensus

        H, W, D = cost.shape
        n = "mccnn_sgm2_band"
        with torch.cuda.device(cost.device):
            rc = adcensus.lib().mccnn_sgm2_band(adcensus._t(imgL, 0, n), adcensus._t(imgR, 0, n), adcensus._t(cost, 0, n),
                                                adcensus._t(acc, 0, n), H, W, D, Ht, Wt, yoff, xoff, opt.pi1, opt.pi2,
                                                opt.tau_so, opt.alpha1, opt.sgm_q1, opt.sgm_q2, int(direction),
                                                int(pass_mask), int(bool(zero_out)), adcensus._stream(cost))
        adcensus._check(rc, "mccnn_sgm2_band")

    def sgm_tables(self, imgL, imgR, D, opt, direction):
        """penalty-class tables + selector words of the full image pair for one `direction` (mccnn_sgm_tables_build)"""
        from . import adcensus

        lib = adcensus.lib()
        Ht, Wt = imgL.shape
        tab = torch.empty(lib.mccnn_sgm_tables_bytes(Ht, Wt, D), dtype=torch.uint8, device=imgL.device)
        n = "mccnn_sgm_tables_build"
        with torch.cuda.device(imgL.device):
            rc = lib.mccnn_sgm_tables_build(adcensus._t(imgL.contiguous(), 0, n), adcensus._t(imgR.contiguous(), 0, n),
                                            tab.data_ptr(), Ht, Wt, D, opt.tau_so, int(direction), adcensus._stream(imgL))
        adcensus._check(rc, "mccnn_sgm_tables_build")
        return tab

    def new_state(self, W, D, like):
        from . import adcensus

        return torch.empty((W, adcensus.lib().mccnn_sgm_state_pitch(D)), device=like.device, dtype=torch.float32)

    def sgm_rows(self, tab, cost, acc, Ht, yoff, opt, direction, pass_mask, zero_out, xa, xb, state_in, state_out):
        from . import adcensus

        H, W, D = cost.shape
        n = "mccnn_sgm2_rows"
        with torch.cuda.device(cost.device):
            rc = adcensus.lib().mccnn_sgm2_rows(tab.data_ptr(), cost.data_ptr(), acc.data_ptr(), H, W, D, int(Ht), int(yoff),
                                                opt.pi1, opt.pi2, opt.tau_so, opt.alpha1, opt.sgm_q1, opt.sgm_q2,
                                                int(direction), int(pass_mask), int(bool(zero_out)), int(xa), int(xb),
                                                adcensus._t(state_in, 0, n, optional=True),
                                                adcensus._t(state_out, 0, n, optional=True), adcensus._stream(cost))
        adcensus._check(rc, "mccnn_sgm2_rows")

    def argmin(self, vol):
        from . import adcensus

        return adcensus.argmin(vol[None])[0, 0]

    def outlier_detection(self, dL, dR, D):
        from . import adcensus

        out = torch.zeros_like(dL)
        adcensus.outlier_detection(dL[None, None], dR[None, None], out[None, None], D)
        return out

    def interpolate_occlusion(self, d, outlier):
        from . import adcensus

        return adcensus.interpolate_occlusion(d[None, None].contiguous(), outlier[None, None].contiguous())[0, 0]

    def interpolate_mismatch(self, d, outlier):
        from . import adcensus

        return adcensus.interpolate_mismatch(d[None, None].contiguous(), outlier[None, None].contiguous())[0, 0]

    def subpixel(self, d_band, vol_band, D):
        from . import adcensus

        return adcensus.subpixel_enchancement(d_band[None, None].contiguous(), vol_band[None].contiguous(), D)[0, 0]

    def median2d(self, d, k):
        from . import adcensus

        return adcensus.median2d(d[None, None].contiguous(), k)[0, 0]

    def mean2d(self, d, sigma, t):
        from . import adcensus

        return adcensus.mean2d(d[None, None].contiguous(), adcensus.gaussian(sigma).to(d.device), t)[0, 0]
