"""Host-side mirror of the feature tower (net_te of main.lua:682-686 / 726-749 at test time): l1 x [3x3 convolution, pad 1]
with ReLU between the layers, Normalize2 at the end for arch 'fast' -- through csrc/feature_tower.cu (layer 1 exact fp32 on
the CUDA cores, the 64 / 112-plane layers as wgmma implicit GEMMs with bf16-split operands).  No fallback.

    tower = FeatureTower(layers, arch="fast")          # [(W (fm, cin, 3, 3), b (fm,)), ...] like cudnn.SpatialConvolution
    feats = tower.forward(x_batch)                     # (2, n_in, H, W) -> (2, fm, H, W): StereoJoin's inputs
"""
import ctypes

import torch

from . import adcensus


class FeatureTower:
    def __init__(self, layers, arch="fast", device=None):
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        ws = [torch.as_tensor(w, dtype=torch.float32).to(self.device).contiguous() for w, _ in layers]
        bs = [torch.as_tensor(b, dtype=torch.float32).reshape(-1).to(self.device).contiguous() for _, b in layers]
        self.fm, self.n_in, self.l1 = ws[0].shape[0], ws[0].shape[1], len(ws)
        if any(tuple(w.shape[2:]) != (3, 3) for w in ws) or any(tuple(w.shape[:2]) != (self.fm, self.fm) for w in ws[1:]):
            raise adcensus.AdcensusError("FeatureTower: expected 3x3 kernels and fm -> fm layers after the first")
        if arch not in ("fast", "slow"):
            raise adcensus.AdcensusError("FeatureTower: arch must be 'fast' (no ReLU after the last layer, Normalize2) or 'slow'")
        relu_last, normalize = (0, 1) if arch == "fast" else (1, 0)
        self._keep = (ws, bs)
        n = len(ws)
        wp = (ctypes.c_void_p * n)(*[w.data_ptr() for w in ws])
        bp = (ctypes.c_void_p * n)(*[b.data_ptr() for b in bs])
        self._h = ctypes.c_void_p()
        stream = torch.cuda.current_stream(self.device).cuda_stream
        adcensus._check(adcensus.lib().mccnn_feature_tower_create(ctypes.byref(self._h), self.n_in, self.fm, self.l1, relu_last,
                                                                  normalize, wp, bp, self.device.index, stream),
                        "mccnn_feature_tower_create")

    def close(self):
        if getattr(self, "_h", None):
            adcensus.lib().mccnn_feature_tower_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, x_batch, nterms=3):
        n = "FeatureTower.forward"
        px = adcensus._t(x_batch, 1, n)
        if x_batch.dim() != 4 or x_batch.shape[1] != self.n_in:
            raise adcensus.AdcensusError("%s: expected (N, %d, H, W)" % (n, self.n_in))
        if x_batch.device != self.device:
            raise adcensus.AdcensusError("%s: input is on %s, the tower's weights on %s" % (n, x_batch.device, self.device))
        N, _, H, W = x_batch.shape
        out = torch.empty((N, self.fm, H, W), device=x_batch.device, dtype=torch.float32)
        with torch.cuda.device(x_batch.device):
            rc = adcensus.lib().mccnn_feature_tower_forward(self._h, px, out.data_ptr(), N, H, W, nterms,
                                                            adcensus._stream(x_batch))
        adcensus._check(rc, n)
        return out
