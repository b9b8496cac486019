"""`TextDetBase` on CUDA tensors: the reference's network seam (basemodel.py:222-244) over the H100 engine.

The reference's `TextDetector` calls `self.net(img_in) -> (blks, mask, lines_map)` with the float32 BGR tensor
`preprocess_img` makes (inference.py:72-83, 146): [N][3][H][W], values in [0, 1], H and W multiples of 64, already on
the model's device.  `TextDetBase` takes that tensor where it is and returns the three outputs as new float32 CUDA
tensors, with the work enqueued on the caller's current stream like any torch op: no copy through the host and no
host synchronisation (`ctd_forward_tensor`).  So

    self.net = ctd_b200.TextDetBase(model_path, device='cuda', act=act); self.backend = 'torch'

puts the engine behind the reference's own `TextDetector.__call__`, whose `non_max_suppression`,
`SegDetectorRepresenter` and the rest run unchanged on the returned tensors.
"""
from pathlib import Path

from . import compiler
from .binding import Engine, PREC_FP16_TC


class TextDetBase:
    """`TextDetBase(model_path, device='cuda', half=False, fuse=False, act='leaky')` (basemodel.py:222-227) and
    `forward(img_in) -> (blks, mask, lines_map)` (basemodel.py:240-244) on the engine.

    model_path: a checkpoint path (the 3-key dict of utils/export.py) or that dict itself.  BatchNorm layers are
    always folded into their convolutions and the network runs in the engine's `precision` (default fp16 tensor
    cores), so `half` and `fuse` are accepted for the reference's signature only.  max_batch and max_size (an int or
    (h, w), multiples of 64) size the engine's workspace: the largest batch and page a call may pass.

    The outputs are float32 CUDA tensors on `device`, fresh per call and without autograd history:
    blks [N][A][5 + nc] (A = 3 * (H/8 * W/8 + H/16 * W/16 + H/32 * W/32), yolo.py:44), mask [N][1][H][W] and
    lines_map [N][2][H][W].  For an input x = u8 / 255 they are bit for bit what `Engine.forward` on the u8 pages
    gives; any other float input is rounded to fp16 in the fp16 engine and used exactly in the fp32 and split ones."""

    def __init__(self, model_path, device='cuda', half=False, fuse=False, act='leaky', precision=None, max_batch=1,
                 max_size=1024):
        import torch
        if isinstance(model_path, (str, Path)):
            if Path(model_path).suffix == '.onnx':
                raise ValueError("%s: an .onnx model is the reference's TextDetBaseDNN (OpenCV-DNN backend); use "
                                 "ctd_b200.TextDetector(model_path) for it" % (model_path,))
            ckpt = torch.load(str(model_path), map_location='cpu')  # reference basemodel.py:212
        else:
            ckpt = model_path
        dev = torch.device(device)
        if dev.type != 'cuda':
            raise ValueError("TextDetBase runs on a CUDA device (there is no CPU fallback), got %s" % (device,))
        self.device = torch.device('cuda', dev.index if dev.index is not None else torch.cuda.current_device())
        if isinstance(max_size, int):
            max_size = (max_size, max_size)
        self.max_size = (int(max_size[0]), int(max_size[1]))
        if self.max_size[0] < 64 or self.max_size[1] < 64 or self.max_size[0] % 64 or self.max_size[1] % 64:
            raise ValueError("max_size sides must be multiples of 64, got %s" % (self.max_size,))
        self.max_batch = int(max_batch)
        if self.max_batch < 1:
            raise ValueError("max_batch must be at least 1, got %d" % self.max_batch)
        self.half, self.fuse = half, fuse
        self.program = compiler.compile_checkpoint(ckpt, head_act=act)
        self.nc = int(getattr(self.program, 'nc', 2))
        # one CUDA graph per (N, H, W), captured on its first call: a loop over same-sized batches pays no launch cost
        self.engine = Engine(self.program, device=self.device.index,
                             precision=PREC_FP16_TC if precision is None else precision, max_batch=self.max_batch,
                             max_h=self.max_size[0], max_w=self.max_size[1], use_graph=True, skip_postproc=True)

    def close(self):
        self.engine.close()

    def _check(self, img_in):
        import torch
        if not isinstance(img_in, torch.Tensor):
            raise ValueError("img_in must be a torch tensor, got %s" % type(img_in).__name__)
        if not img_in.is_cuda or img_in.device.index != self.device.index:
            raise ValueError("img_in must be on %s, got %s" % (self.device, img_in.device))
        if img_in.dtype != torch.float32:
            raise ValueError("img_in must be float32, got %s" % img_in.dtype)
        if img_in.dim() != 4 or img_in.shape[1] != 3:
            raise ValueError("img_in must be [N][3][H][W], got %s" % (tuple(img_in.shape),))
        n, _, h, w = img_in.shape
        if n < 1 or n > self.max_batch:
            raise ValueError("batch of %d: this module takes 1 to max_batch = %d pages" % (n, self.max_batch))
        if h < 64 or w < 64 or h % 64 or w % 64 or h > self.max_size[0] or w > self.max_size[1]:
            raise ValueError("page %dx%d: H and W must be multiples of 64 and at most max_size %dx%d"
                             % (h, w, self.max_size[0], self.max_size[1]))

    def forward(self, img_in):
        """img_in: float32 [N][3][H][W] BGR on this module's device -> (blks, mask, lines_map), enqueued on the
        device's current stream.  Raises ValueError, before any GPU work, for any other tensor."""
        import torch
        self._check(img_in)
        n, _, h, w = img_in.shape
        x = img_in.detach().contiguous()
        if x.data_ptr() % 16:   # the pre-pass reads four pixels per 16-byte load
            x = x.clone()
        rows = 3 * ((h // 8) * (w // 8) + (h // 16) * (w // 16) + (h // 32) * (w // 32))
        stream = torch.cuda.current_stream(self.device)
        blks = torch.empty((n, rows, 5 + self.nc), dtype=torch.float32, device=self.device)
        mask = torch.empty((n, 1, h, w), dtype=torch.float32, device=self.device)
        lines = torch.empty((n, 2, h, w), dtype=torch.float32, device=self.device)
        self.engine.forward_tensor(x.data_ptr(), n, h, w, stream.cuda_stream, blks.data_ptr(), mask.data_ptr(),
                                   lines.data_ptr())
        return blks, mask, lines

    __call__ = forward
