"""torchvision ResNet50 court-keypoint regressor on the project's CUDA kernels: the `model_type="resnet"` branch of
/root/reference/trackers/keypoints_tracker/keypoints_tracker.py:158-167 (model: resnet50 with fc -> 2 * 12 outputs),
:276-312 (forward, sigmoid, scaling by the frame size) and keypoints_tracker/iterable.py:10-41 (BGR -> RGB, PIL
Resize((224, 224)) = Image.BILINEAR, ToTensor, Normalize).

Layers: pre-processing (Pillow-exact bilinear resize on device, normalise), conv1 7x7/s2 + maxpool (CUDA cores,
csrc/resnet_aux.cu), the 16 bottlenecks as 52 fused conv launches on the wgmma conv kernels (BN folded, identity added
before the ReLU in the epilogue, 1x1 stride-2 downsample convs), global average pool + fc + sigmoid.
State-dict key names are torchvision's (`layer1.0.conv1.weight`, `fc.weight`, ...), so real checkpoints load.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _lib as L
from . import ops, resample

MEAN = (0.485, 0.465, 0.406)  # sic: the reference's green mean is 0.465, not ImageNet's 0.456 (iterable.py:22)
STD = (0.229, 0.224, 0.225)
SIZE = 224
_LAYERS = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))  # planes, blocks, stride of the first block


def _fold(sd, conv, bn, eps=1e-5):
    return ops.fold_bn(sd[f"{conv}.weight"].float(), sd[f"{bn}.weight"].float(), sd[f"{bn}.bias"].float(),
                       sd[f"{bn}.running_mean"].float(), sd[f"{bn}.running_var"].float(), eps)


class ResNet50Engine:
    """`model(x)` surface of the reference plus a fused `predict_frames(frames_bgr) -> (n, n_out) float32 sigmoid`."""

    def __init__(self, state_dict: dict, max_batch: int = 8, device: str = "cuda"):
        if not torch.cuda.is_available():
            raise L.PbError("ResNet50Engine needs a CUDA device (no CPU fallback)")
        L.lib()
        self.device = torch.device(device)
        self.B = max_batch
        sd = state_dict
        self.n_out = sd["fc.weight"].shape[0]
        dev, B = self.device, self.B
        h = lambda hh, ww, c: torch.zeros((B, hh, ww, c), dtype=torch.float16, device=dev)
        self.x_in = torch.zeros((B, SIZE, SIZE, 4), dtype=torch.float16, device=dev)
        self.c1 = h(112, 112, 64)
        self.p1 = h(56, 56, 64)
        w, b = _fold(sd, "conv1", "bn1")  # (64,3,7,7) -> [(r*7+s)*3+c][64]
        self.w_stem = w.permute(2, 3, 1, 0).reshape(147, 64).contiguous().to(dev)
        self.b_stem = b.contiguous().to(dev)
        self.fc_w = sd["fc.weight"].float().contiguous().to(dev)
        self.fc_b = sd["fc.bias"].float().contiguous().to(dev)
        self.out = torch.zeros((B, self.n_out), dtype=torch.float32, device=dev)
        P = ops.Program()
        self._keep = []
        R = L.ACT_RELU

        def conv(x, cin, conv_name, bn_name, out, k, s, act, res=None):
            w, b = _fold(sd, conv_name, bn_name)
            cout = w.shape[0]
            wp, bp = ops.pack_conv_weight(w, b, cin, ops.pad16(cout), dev)
            self._keep += [wp, bp]
            P.conv(ops.make_conv_desc(x, 0, cin, wp, bp, k, s, act, out, 0, L.OUT_F16_NHWC, None, res, 0,
                                      res_before_act=res is not None), cin_real=w.shape[1], cout_real=cout)

        x, cin, hw = self.p1, 64, 56
        for li, (planes, blocks, stride) in enumerate(_LAYERS, start=1):
            for bi in range(blocks):
                s = stride if bi == 0 else 1
                ho = hw // s
                pre = f"layer{li}.{bi}"
                t1, t2, o = h(hw, hw, planes), h(ho, ho, planes), h(ho, ho, 4 * planes)
                self._keep += [t1, t2, o]
                conv(x, cin, f"{pre}.conv1", f"{pre}.bn1", t1, 1, 1, R)
                conv(t1, planes, f"{pre}.conv2", f"{pre}.bn2", t2, 3, s, R)  # torchvision v1.5: stride on the 3x3
                if f"{pre}.downsample.0.weight" in sd:
                    idt = h(ho, ho, 4 * planes)
                    self._keep.append(idt)
                    conv(x, cin, f"{pre}.downsample.0", f"{pre}.downsample.1", idt, 1, s, L.ACT_NONE)
                else:
                    idt = x
                conv(t2, planes, f"{pre}.conv3", f"{pre}.bn3", o, 1, 1, R, res=idt)
                x, cin, hw = o, 4 * planes, ho
        self.feat, self.feat_hw, self.feat_c = x, hw * hw, cin
        self.prog = P
        self._mean = (C.c_float * 3)(*MEAN)
        self._std = (C.c_float * 3)(*STD)
        self._tables = {}
        self._stage = None
        self._host = [torch.zeros((B, self.n_out), dtype=torch.float32).pin_memory() for _ in range(3)]
        self._turn = 0

    def to(self, device):
        return self

    def eval(self):
        return self

    # ---- stages ----------------------------------------------------------------------------------------------
    def _forward_from_input(self, n: int):
        """self.x_in[:n] (normalised fp16 pixels) -> self.out[:n] (sigmoid of the fc output)."""
        lib, st = L.lib(), L.stream_ptr()
        L.check(lib.pb_resnet_stem7x7(self.x_in.data_ptr(), self.B, SIZE, SIZE, self.w_stem.data_ptr(),
                                      self.b_stem.data_ptr(), self.c1.data_ptr(), st))
        L.check(lib.pb_maxpool3x3s2(self.c1.data_ptr(), self.B, 112, 112, 64, self.p1.data_ptr(), st))
        self.prog.run()
        L.check(lib.pb_avgpool_fc_sigmoid(self.feat.data_ptr(), self.B, self.feat_hw, self.feat_c, self.fc_w.data_ptr(),
                                          self.fc_b.data_ptr(), self.n_out, self.out.data_ptr(), st))

    @torch.no_grad()
    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        """Reference-compatible call (keypoints_tracker.py:296): NCHW fp32 normalised batch -> (n, n_out) LOGITS are
        not kept by the fused tail; this returns logit(sigmoid) so that `torch.nn.Sigmoid()(model(x))` reproduces the
        engine's output exactly."""
        n = x.shape[0]
        if n > self.B or tuple(x.shape[1:]) != (3, SIZE, SIZE):
            raise L.PbError(f"ResNet50Engine: expected (<= {self.B}, 3, {SIZE}, {SIZE}), got {tuple(x.shape)}")
        self.x_in[:n, ..., :3] = x.to(self.device).permute(0, 2, 3, 1).to(torch.float16)
        self._forward_from_input(n)
        p = self.out[:n].clone().clamp(1e-7, 1 - 1e-7)
        return torch.log(p) - torch.log1p(-p)

    @torch.no_grad()
    def predict_frames(self, frames) -> np.ndarray:
        """frames: list of HWC uint8 BGR arrays or a uint8 (n,H,W,3) tensor (host or device), n <= max_batch.
        BGR -> RGB, Pillow-exact bilinear resize to 224 x 224, ToTensor + Normalize, network, sigmoid.
        Returns (n, n_out) float32 on the host."""
        t = frames if isinstance(frames, torch.Tensor) else torch.from_numpy(np.stack([np.ascontiguousarray(f) for f in frames]))
        if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[-1] != 3:
            raise L.PbError("frames must be uint8 (n,H,W,3)")
        n, Hs, Ws, _ = t.shape
        if n > self.B:
            raise L.PbError(f"batch {n} exceeds engine max_batch {self.B}")
        if t.device.type != "cuda":
            if self._stage is None or self._stage.shape[1:] != t.shape[1:]:
                self._stage = torch.empty((self.B,) + tuple(t.shape[1:]), dtype=torch.uint8, device=self.device)
            self._stage[:n].copy_(t, non_blocking=True)
            t = self._stage[:n]
        t = t.contiguous()
        key = (Hs, Ws)
        if key not in self._tables:
            bh, kh, ksh = resample.pil_bilinear_tables(Ws, SIZE)
            bv, kv, ksv = resample.pil_bilinear_tables(Hs, SIZE)
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)
            self._tables[key] = dict(bh=up(bh), kh=up(kh), ksh=ksh, bv=up(bv), kv=up(kv), ksv=ksv,
                                     tmp=torch.empty((self.B, Hs, SIZE, 3), dtype=torch.uint8, device=self.device),
                                     small=torch.empty((self.B, SIZE, SIZE, 3), dtype=torch.uint8, device=self.device))
        tb = self._tables[key]
        lib, st = L.lib(), L.stream_ptr()
        L.check(lib.pb_pil_resize_u8(t.data_ptr(), n, Hs, Ws, tb["tmp"].data_ptr(), tb["small"].data_ptr(), SIZE, SIZE,
                                     tb["bh"].data_ptr(), tb["kh"].data_ptr(), tb["ksh"], tb["bv"].data_ptr(),
                                     tb["kv"].data_ptr(), tb["ksv"], 1, None, 0, st))
        L.check(lib.pb_u8_normalize_f16(tb["small"].data_ptr(), n * SIZE * SIZE, self._mean, self._std,
                                        self.x_in.data_ptr(), st))
        self._forward_from_input(n)
        host = self._host[self._turn]
        self._turn = (self._turn + 1) % len(self._host)
        host[:n].copy_(self.out[:n], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return host[:n].numpy().copy()
