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

Where a band's cost volumes come from (:func:`band_source`): :func:`stereo_predict_rowband` takes the replicated
'fast' features; :func:`band_predict` / :func:`predict_pair` start from the two standardised images, replicated, and run
the feature tower (and the 'slow' scorer head) or census / AD on the band's rows only.  The 'fast', 'ad' and 'census'
volumes are cheap, so they cover the extended band of the first CBCA block as above.  The 'slow' head dominates the
pair's time, so each pixel is scored on exactly one rank and the first block exchanges its halo rows like the second.
"""
import math
import os

import numpy as np
import torch
import torch.distributed as dist

from . import pipeline


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

    def barrier(self):
        if self.on:
            dist.barrier()


def _refuse_stage_options(opt):
    for k in ("sm_terminate", "sm_skip"):
        if getattr(opt, k, 0):
            raise ValueError("row-band stereo_predict runs the full chain only: -%s is not supported (use the "
                             "single-GPU pipeline)" % k)


def stereo_predict_rowband(ops, featL, featR, imgL, imgR, D, opt, comm=None, chunks=None):
    """main.lua:929-1082 (arch 'fast') with the rows of one pair split over the ranks of `comm`.

    featL/featR (C,H,W) and imgL/imgR (H,W) are the FULL tensors on every rank (only this rank's
    rows of the features are read).  `chunks`: column chunks of the vertical SGM wavefront (default: 4 per rank, at
    least 32 columns each).  Returns the full (H,W) disparity map on every rank.  Only the full chain: parameters with
    ``sm_terminate`` / ``sm_skip`` set are refused before any work (run them on one GPU through the fused pipeline).
    """
    _refuse_stage_options(opt)

    def join(a, b, dirs):
        volL, volR = ops.stereo_join(featL[:, a:b].contiguous(), featR[:, a:b].contiguous(), D)   # :946-947
        ops.fix_border(volL, opt.border, -1)                                                     # :948
        ops.fix_border(volR, opt.border, 1)                                                      # :949
        return volL, volR

    return band_chain(ops, join, True, imgL, imgR, D, opt, comm, chunks)


def band_source(ops, x_batch, D, opt, arch, tower=None, head=None):
    """The cost volumes of image rows [a, b) of one pair, as main.lua:929-981 holds them at :986 (NaN fill, fix_border
    applied), without computing the volumes of any other row.

    x_batch (2,1,H,W): the two standardised images (left, right), whole.  arch 'fast' / 'slow' take `tower` (an object
    with ``forward((2,1,h,W)) -> (2,fm,h,W)`` and ``l1`` 3x3 layers: :class:`feature_tower.FeatureTower`) and for 'slow'
    `head` (``volumes(fL, fR, D, want_left=, want_right=)``: :class:`scorer_head.ScorerHead`).  The tower runs on the rows
    [a - l1, b + l1) and keeps [a, b): every pixel it keeps is then as far from the crop's zero padding as the tower
    reaches; census / AD (9 x 9 windows) likewise run on [a - 4, b + 4).

    Returns (volumes, extends): volumes(a, b, dirs) -> (volL, volR), each (D, b - a, W) or None when its direction
    (-1 left, 1 right) is not in `dirs` and skipping it saves work; `extends` says whether the volumes of a row are cheap
    enough to compute again on the neighbouring bands ('fast', 'ad', 'census': the first CBCA block then runs on the
    extended band) or not ('slow': every row is scored by exactly one rank, the first block exchanges halo rows)."""
    pipeline.check_arch(arch)
    H = x_batch.shape[2]

    def rows(a, b, m):
        """image rows [a - m, b + m) clipped to the image, and where row a lies in them"""
        a0, b0 = max(0, a - m), min(H, b + m)
        return x_batch[:, :, a0:b0].contiguous(), a - a0

    if arch in ("ad", "census"):
        cost = ops.census if arch == "census" else ops.ad

        def volumes(a, b, dirs):
            x, o = rows(a, b, 4)
            vl = cost(x[0], x[1], D, -1)[:, o:o + b - a].contiguous() if -1 in dirs else None   # :934 / :940
            vr = cost(x[1], x[0], D, 1)[:, o:o + b - a].contiguous() if 1 in dirs else None     # :935 / :941
            return vl, vr

        return volumes, True
    if tower is None or (arch == "slow" and head is None):
        raise ValueError("arch '%s' needs the feature tower%s" % (arch, " and the scorer head" if arch == "slow" else ""))

    def volumes(a, b, dirs):
        x, o = rows(a, b, int(tower.l1))
        f = tower.forward(x)                                                                  # :944 / :957
        fL, fR = f[0, :, o:o + b - a].contiguous(), f[1, :, o:o + b - a].contiguous()
        del f
        if arch == "fast":
            vl, vr = ops.stereo_join(fL, fR, D)                                               # :946-947
        else:
            vl, vr = head.volumes(fL, fR, D, want_left=-1 in dirs, want_right=1 in dirs)      # :962-979
            vl, vr = (v[0] if v is not None else None for v in (vl, vr))
        if vl is not None:
            ops.fix_border(vl, opt.border, -1)                                                # :948 / :981
        if vr is not None:
            ops.fix_border(vr, opt.border, 1)
        return vl, vr

    return volumes, arch == "fast"


def band_predict(ops, x_batch, D, opt, arch, tower=None, head=None, comm=None, chunks=None, want_vols=False):
    """main.lua:929-1082 for any architecture, from the standardised images (2,1,H,W) (whole, on every rank) with the rows
    split over the ranks of `comm`: each rank computes the cost volumes of its own band only (:func:`band_source`).

    Returns the full (H,W) disparity map on every rank; with `want_vols` also this rank's rows [y0, y1) = split(H, N, r) of
    the left and right volumes after the chain (D, y1 - y0, W), both directions computed even without the LR check, as
    main.lua's -a predict writes both (main.lua:1042-1047)."""
    _refuse_stage_options(opt)
    volumes, extends = band_source(ops, x_batch, D, opt, arch, tower, head)
    return band_chain(ops, volumes, extends, x_batch[0, 0], x_batch[1, 0], D, opt, comm, chunks, want_vols)


def cbca_halo(opt):
    """(max_arm, halo): the longest cross arm max(L1, 2), and the rows one CBCA iteration reaches into a neighbouring band
    (0 without CBCA)"""
    max_arm = max(int(opt.L1), 2)
    return max_arm, (max_arm - 1 if (opt.cbca_i1 + opt.cbca_i2) > 0 else 0)


def source_rows(H, world, rank, opt, extends):
    """[ya, yb): the rows whose cost volumes rank `rank` of `world` computes -- its band split(H, world, rank), extended by
    cbca_i1 * halo rows on either side (clipped to the image) when the volume source `extends`"""
    y0, y1 = split(H, world, rank)
    e1 = cbca_halo(opt)[1] * int(opt.cbca_i1) if extends else 0
    return max(0, y0 - e1), min(H, y1 + e1)


def band_chain(ops, volumes, extends, imgL, imgR, D, opt, comm=None, chunks=None, want_vols=False):
    """The chain of main.lua:986-1082 on this rank's band from `volumes(a, b, dirs)` (see :func:`band_source`).  With
    `extends` the first CBCA block runs on the band extended by cbca_i1 * halo rows, whose volumes are computed here too;
    otherwise on the band itself, with the halo rows exchanged with the neighbours."""
    comm = comm or Comm()
    H, W = imgL.shape
    N, r = comm.world, comm.rank
    y0, y1 = split(H, N, r)
    Hb = y1 - y0
    max_arm, halo = cbca_halo(opt)
    band_min = min(split(H, N, p)[1] - split(H, N, p)[0] for p in range(N))
    if N > 1:
        assert band_min >= max(halo, 1), "bands thinner than the CBCA halo"
        assert max_arm <= 14, "row-band CBCA supports arms up to 14 pixels"
    # column chunks of the vertical wavefront: a chunk's scan is latency-bound (Hb serial steps) unless it is wide, and the chain
    # costs (N - 1 + K) chunk times: K = N is the measured sweet spot (K = 4 N made 39 hops of 94 columns at Middlebury size)
    K = chunks if chunks else max(1, min(N, W // 32)) if N > 1 else 1

    # first CBCA block on the band extended by cbca_i1 * halo rows when the volume source covers the extension (features or
    # images are replicated), else on the band with an exchange
    ya, yb = source_rows(H, N, r, opt, extends)
    # main.lua:954-955: without the LR check (mb) only direction -1 is consumed, unless the volumes are asked for
    dirs = (1, -1) if (opt.lr_check or want_vols) else (-1,)
    src = dict(zip((-1, 1), volumes(ya, yb, dirs)))                                                  # :929-981
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
    band_vols = {}
    for direction in dirs:                                                                           # :955
        ext = src.pop(direction)                                                                     # :986
        if extends:
            ext = cbca_block(ext, ya, yb, int(opt.cbca_i1), direction)                               # :998-1001
            vol = ext[:, y0 - ya: y0 - ya + Hb].contiguous() if (ya != y0 or yb != y1) else ext
        else:
            vol = cbca_exchanging(ext, int(opt.cbca_i1), direction)
        del ext
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
        if want_vols or direction == -1:
            band_vols[direction] = vol
    vol_left = band_vols[-1]

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
    d = band_filter(lambda t: ops.mean2d(t, opt.blur_sigma, opt.blur_t), d, kr)                      # :1078
    return (d, band_vols[-1], band_vols[1]) if want_vols else d


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

    def _image_cost(self, fn, x0, x1, D, direction):
        """x0, x1 (nch, h, W) -> the (D, h, W) volume of adcensus.ad / census on a NaN-filled tensor (main.lua:933-941)"""
        from . import adcensus

        out = torch.empty((1, D) + tuple(x0.shape[1:]), device=x0.device, dtype=torch.float32)
        adcensus.fill_nan(out)
        fn(x0[None].contiguous(), x1[None].contiguous(), out, direction)
        return out[0]

    def ad(self, x0, x1, D, direction):
        from . import adcensus

        return self._image_cost(adcensus.ad, x0, x1, D, direction)

    def census(self, x0, x1, D, direction):
        from . import adcensus

        return self._image_cost(adcensus.census, x0, x1, D, direction)

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


def write_outputs(out_dir, disp, volL, volR, comm=None):
    """right.bin and left.bin ((1, D, H, W) raw little-endian fp32, main.lua:1042-1047) and disp.bin ((1, 1, H, W), :1103)
    from what each rank holds: `disp` (H, W), the same on every rank, and this rank's rows [y0, y1) of the two volumes
    (D, y1 - y0, W).  Rank 0 creates the files at their full size; then every rank writes its rows of each disparity plane
    at their offsets (D writes of (y1 - y0) x W floats per volume).  No volume crosses a GPU: each rank copies its own band
    to the host and nothing else.  The ranks must share `out_dir` (one node, or a shared file system)."""
    comm = comm or Comm()
    H, W = disp.shape
    D = volL.shape[0]
    y0, y1 = split(H, comm.world, comm.rank)
    files = (("right.bin", volR), ("left.bin", volL))                  # direction 1 comes first
    if comm.rank == 0:
        os.makedirs(out_dir, exist_ok=True)
        for name, _ in files:
            with open(os.path.join(out_dir, name), "wb") as f:
                f.truncate(D * H * W * 4)
    comm.barrier()
    for name, v in files:
        a = np.ascontiguousarray(v.cpu().numpy() if isinstance(v, torch.Tensor) else v, dtype="<f4")
        assert a.shape == (D, y1 - y0, W), "volume rows %s, expected %s" % (a.shape, (D, y1 - y0, W))
        fd = os.open(os.path.join(out_dir, name), os.O_WRONLY)
        try:
            for d in range(D):
                os.pwrite(fd, a[d].tobytes(), (d * H + y0) * W * 4)
        finally:
            os.close(fd)
    if comm.rank == 0:
        d = np.ascontiguousarray(disp.cpu().numpy() if isinstance(disp, torch.Tensor) else disp, dtype="<f4")
        d.tofile(os.path.join(out_dir, "disp.bin"))
    comm.barrier()


def predict_pair(left=None, right=None, dataset="kitti", arch="census", disp_max=70, x_batch=None, net_fname=None,
                 tower=None, head=None, comm=None, device=None, out_dir=None, want_vols=False, chunks=None, **overrides):
    """``main.lua <dataset> <arch> -a predict`` (:func:`frontend.predict`) with the rows of the pair split over the ranks of
    `comm`, one GPU per rank (`device`: a torch.device or index, default the current device).

    The pair: the image files (or arrays) `left` / `right`, standardised on every rank as :func:`frontend.make_batch` does,
    or the standardised batch `x_batch` (2,1,H,W).  arch 'fast' / 'slow' take the network from `net_fname` (the reference's
    ascii .t7), or the stages `tower` (and for 'slow' `head`) built on this rank's device; 'ad' / 'census' need neither.
    `overrides` are the stereo method's options (pipeline.make_params); -sm_terminate / -sm_skip are refused.

    With `out_dir`, writes right.bin, left.bin and disp.bin there (:func:`write_outputs`): the bytes frontend.predict writes
    for the same images, dataset, arch, network, disp_max and overrides.  Returns the disparity map (H, W) float32 numpy on
    every rank; with `want_vols` also this rank's rows of the left and right volumes, (D, y1 - y0, W) device tensors.
    Every check on the arguments and the network file is made before any GPU work."""
    from . import frontend

    method = frontend.StereoMethod(dataset, arch, None if tower is not None else net_fname, **overrides)
    _refuse_stage_options(method.opt)
    if method.needs_net and tower is None:
        raise ValueError("arch '%s' needs -net_fname (or the stage objects `tower` / `head`)" % arch)
    if arch == "slow" and tower is not None and head is None:
        raise ValueError("arch 'slow' needs the scorer head with the feature tower")
    if x_batch is None:
        x_batch = frontend.make_batch(left, right)                                   # main.lua:1085-1100
    D = int(disp_max)
    dev = device if isinstance(device, torch.device) else \
        torch.device("cuda", torch.cuda.current_device() if device is None else device)
    comm = comm or Comm()
    with torch.cuda.device(dev):
        xb = torch.as_tensor(x_batch, dtype=torch.float32).to(dev).contiguous()
        if xb.dim() != 4 or xb.shape[:2] != (2, 1):
            raise ValueError("x_batch: (2, 1, H, W) expected, got %s" % (tuple(xb.shape),))
        try:
            if tower is None:
                tower, head = method.stages(dev)
            vols = want_vols or out_dir is not None
            out = band_predict(CudaOps(dev), xb, D, method.opt, arch, tower, head, comm, chunks, want_vols=vols)
            disp, volL, volR = out if vols else (out, None, None)
        finally:
            method.close()
        disp_h = disp.cpu().numpy()
        if out_dir is not None:
            write_outputs(out_dir, disp_h, volL, volR, comm)
    return (disp_h, volL, volR) if want_vols else disp_h
