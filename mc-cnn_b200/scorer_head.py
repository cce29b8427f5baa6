"""Host-side mirror of the accurate ('slow') architecture's scorer head: net_te2 of main.lua:688-695 applied per disparity
(main.lua:958-984) -- through the fused wgmma kernel of csrc/scorer_head.cu.  No fallback: the call raises if the CUDA
library is missing.

    head = ScorerHead(layers)                 # [(W (out, in), b (out,)), ...] as in net_te2: l2 hidden layers + (1, nh2)
    volL, volR = head.volumes(featL, featR, D)  # (1, D, H, W) each, NaN where the reference leaves its fill (:962)

`layers` follows the modules of net_te2 (SpatialConvolution1_fw: weight (out, in), bias (1, out, 1, 1)).
"""
import ctypes

import torch

from . import adcensus


class ScorerHead:
    def __init__(self, layers, device=None):
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        ws, bs = [], []
        for w, b in layers:
            ws.append(torch.as_tensor(w, dtype=torch.float32).to(self.device).contiguous())
            bs.append(torch.as_tensor(b, dtype=torch.float32).reshape(-1).to(self.device).contiguous())
        self.l2 = len(ws) - 1
        self.nh2 = ws[0].shape[0]
        if ws[0].shape[1] % 2 or ws[-1].shape != (1, self.nh2) or any(w.shape != (self.nh2, self.nh2) for w in ws[1:-1]):
            raise adcensus.AdcensusError("ScorerHead: layer shapes do not form net_te2 (2 fm -> nh2 -> ... -> nh2 -> 1)")
        self.fm = ws[0].shape[1] // 2
        self._keep = (ws, bs)
        n = len(ws)
        wp = (ctypes.c_void_p * n)(*[w.data_ptr() for w in ws])
        bp = (ctypes.c_void_p * n)(*[b.data_ptr() for b in bs])
        self._h = ctypes.c_void_p()
        lib = adcensus.lib()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        adcensus._check(lib.mccnn_scorer_head_create(ctypes.byref(self._h), self.fm, self.nh2, self.l2, wp, bp,
                                                     self.device.index, stream), "mccnn_scorer_head_create")

    def close(self):
        if getattr(self, "_h", None):
            adcensus.lib().mccnn_scorer_head_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def volumes(self, featL, featR, D, nterms=3, want_left=True, want_right=True):
        """featL / featR: (fm, H, W) tower outputs (left / right image).  Returns (volL, volR), each (1, D, H, W) or None:
        volL[0, d, :, d:] = volR[0, d, :, :W-d] = the head's score of disparity d (main.lua:963-978), NaN elsewhere."""
        n = "ScorerHead.volumes"
        pL, pR = adcensus._t(featL, 1, n), adcensus._t(featR, 2, n)
        if featL.dim() != 3 or featL.shape != featR.shape or featL.shape[0] != self.fm:
            raise adcensus.AdcensusError("%s: expected two (%d, H, W) tensors" % (n, self.fm))
        if featL.device != self.device or featR.device != self.device:
            raise adcensus.AdcensusError("%s: features are on %s and %s, the head's weights on %s"
                                         % (n, featL.device, featR.device, self.device))
        _, H, W = featL.shape
        vols = []
        for want in (want_left, want_right):
            vols.append(torch.full((1, D, H, W), float("nan"), device=featL.device) if want else None)   # main.lua:962
        with torch.cuda.device(featL.device):
            rc = adcensus.lib().mccnn_scorer_head_forward(self._h, pL, pR, adcensus._t(vols[0], 0, n, optional=True),
                                                          adcensus._t(vols[1], 0, n, optional=True), H, W, D, nterms,
                                                          adcensus._stream(featL))
        adcensus._check(rc, n)
        return vols[0], vols[1]
