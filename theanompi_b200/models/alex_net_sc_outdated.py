"""``AlexNet_sc`` (ref ``alex_net_sc_outdated.py``): AlexNet with mean Subtract + random Crop
*inside* the step instead of in the loader (O8)."""
from __future__ import annotations

from .alex_net import AlexNet
from .layers2 import Crop, Subtract, forward_chain


class AlexNet_sc(AlexNet):
    graph_safe = False            # the in-graph Crop layer draws offsets / mirrors from the host RNG every step
    supports_mixup = False        # the outdated in-step Subtract / Crop variant of AlexNet
    supports_model_ema = False    # the outdated variant: the average is offered on the loader-fed AlexNet
    supports_sam = False          # its in-graph Crop draws new crops at every forward: a second forward would see another crop
    supports_resized_crop = False  # its crop is the in-graph Crop layer, not the loader's
    supports_distill = False       # its in-graph Crop: the teacher would see the uncropped batch
    def __init__(self, config):
        config = dict(config)
        config["no_paraload"] = True
        super().__init__(config)
        self.name = "AlexNet_sc"
        B = self.batch_size
        self.sub = Subtract(input=None, input_shape=(B, self.data.height, self.data.width, self.channels),
                            subtract_arr=self.data.rawdata[4] / 255.0, printinfo=False)
        self.crop = Crop(input=self.sub, output_shape=(B, self.input_height, self.input_width, self.channels),
                         flag_batch=self.batch_crop_mirror, printinfo=False)
        import torch
        full = (self.file_batch_size, self.data.height, self.data.width, self.channels)
        self.shared_x = torch.zeros(full, dtype=self.act_dtype, device=self.device)
        self.x_in = torch.zeros((B,) + full[1:], dtype=self.act_dtype, device=self.device)

    def forward(self, x):
        return forward_chain(self.layers, self.crop.forward(self.sub.forward(x)))

    def _load_file_batch(self, mode, idx, img, labels, n_batches):
        import numpy as np
        import torch
        raw = np.empty((self.file_batch_size, self.data.height, self.data.width, self.channels), dtype=np.uint8)
        src = self.data.read(img[idx], raw)
        t = src if src is not None else torch.from_numpy(raw)
        if self.cuda:
            t = (t if t.is_pinned() else t.pin_memory()).to(self.device, non_blocking=True)
        self.shared_x.copy_(t.to(self.act_dtype) / 255.0)
        self._labels_to_device(labels[idx])
        return idx == n_batches - 1
