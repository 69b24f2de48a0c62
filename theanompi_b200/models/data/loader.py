"""Parallel data loader (H100-native replacement of ``proc_load_mpi.py``).

Reference mechanism (``theanompi/models/data/proc_load_mpi.py:16-133``,
``imagenet.py:226-321``): an ``MPI.COMM_SELF.Spawn``-ed child process per worker
loads an ``.hkl`` file, normalises / crops / mirrors it on the CPU in fp32, uploads
it from pageable memory into its own GPU buffer, and copies it into the trainer's
``shared_x`` through a CUDA-IPC handle obtained over ZeroMQ; double buffering is
implicit in the tag-40 / tag-55 message protocol.

Here the same producer/consumer contract (``request(next file)`` … ``get()`` blocks
until that batch sits in the trainer's input buffer) is built from:

* a loader **thread** (file IO / numpy release the GIL) filling **pinned** host ring
  slots with the raw uint8 NHWC batch,
* ``cudaMemcpyAsync`` H2D of the uint8 payload on a dedicated **copy stream**
  (4× fewer PCIe bytes than the reference's cropped fp32),
* one fused device kernel (``csrc/data_kernels.cu``): (x − mean)·scale → random crop →
  mirror → bf16 NHWC, straight into the slot the model reads,
* CUDA events for both directions of the hand-off (ready → trainer stream waits;
  consumed → the loader may overwrite the slot), so neither side ever blocks the
  host on GPU work.

On CPU (tests) the same class runs synchronously with the numpy reference.
"""
from __future__ import annotations

import queue
import threading

import numpy as np
import torch

from ... import ops
from .utils import (AA_RECORD_FLOATS, CJ_RECORD_FLOATS, aa_bilinear, aa_slots, augmix_records, auto_augment_records, auto_augment_rng,
                    color_jitter_records, color_jitter_rng, draw_crops, draw_erase_boxes, draw_resized_crops, random_erasing_rng,
                    resized_crop_rng)


class LoadedBatch(object):
    """One loaded batch; ``boxes`` / ``flips``: the host copies of the random-resized-crop draw it was made with, or of the fixed
    crops as boxes of the output's size under colour jitter (None otherwise); ``records``: the colour-jitter records (None otherwise);
    ``erase``: the random-erasing boxes (i, j, h, w) in output coordinates (None otherwise); ``aa_records``: the auto_augment op
    records, float32 [N, slots, 12] (None otherwise); ``aa_weights``: AugMix's mixing weights, float32 [N, 1 + width] (None
    otherwise)."""
    __slots__ = ("x", "slot", "ready", "item", "h2d_bytes", "boxes", "flips", "records", "erase", "aa_records", "aa_weights")

    def __init__(self, x, slot, ready, item, h2d_bytes, boxes=None, flips=None, records=None, erase=None, aa_records=None,
                 aa_weights=None):
        self.x, self.slot, self.ready, self.item, self.h2d_bytes = x, slot, ready, item, h2d_bytes
        self.boxes, self.flips, self.records, self.erase, self.aa_records = boxes, flips, records, erase, aa_records
        self.aa_weights = aa_weights


class ParaLoader(object):
    def __init__(self, read_fn, device, raw_shape, crop_hw, mean, std_scale=1.0 / 255.0,
                 out_dtype=None, depth=2, rand_crop=True, batch_crop_mirror=False, seed=1234,
                 threaded=True, host_buffers=None, on_close=None, resized_crop=None, rank=0, color_jitter=None,
                 random_erasing=None, auto_augment=None, val_crops=1):
        """``resized_crop``: a validated ``config['random_resized_crop']`` (``utils.check_resized_crop``) or None; with it every
        "train" batch is a random-resized crop drawn per image from the generator keyed by (its seed, ``rank``), and "val" batches
        keep the centre crop.  ``color_jitter``: a validated ``config['color_jitter']`` (``utils.check_color_jitter``) or None; with
        it every "train" image gets a colour map drawn from the generator keyed by (its seed, ``rank``, 1), applied by the crop
        kernel on the same boxes or fixed crops as without it; "val" batches are never jittered.  ``random_erasing``: a validated
        ``config['random_erasing']`` (``utils.check_random_erasing``) or None; with it every "train" batch, whichever crop path made
        it, gets erase boxes drawn from the generator keyed by (its seed, ``rank``, 3) and zeroed in the output slot by one more
        launch on the copy stream; "val" batches are never erased.  ``auto_augment``: a validated ``config['auto_augment']``
        (``utils.check_auto_augment``) or None; with it every "train" image gets TrivialAugmentWide / RandAugment / AutoAugment / AugMix
        op records (and AugMix's mixing weights) drawn from the generator keyed by (its seed, ``rank``, 2), applied on the uint8 crop of
        the same boxes or fixed crops between the crop and the normalisation; "val" batches are never augmented.  Only "augmix"
        allocates the chains' uint8 ping-pong pairs (2 × width crops) and the weight records.  ``val_crops``: 1, 2 or 10 (``utils.check_val_crops``); with
        V > 1 every "val" batch is the view-major [V, N, ch, cw, C] of ``multi_crop_norm`` (``reference.multi_crop_views``), cut by one
        launch from the staged uint8 batch into a ring of its own (10 × 128 × 227² × 3 × 2 B ≈ 396 MB per slot in bf16, twice that in
        fp32, times ``depth``, allocated only when V > 1); "train" batches, their slots and draws do not change."""
        self.read_fn = read_fn
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        self.raw_shape = tuple(raw_shape)
        self.crop_hw = tuple(crop_hw)
        self.depth = depth
        self.rand_crop, self.batch_crop_mirror = rand_crop, batch_crop_mirror
        self.mode = "train"
        self.rs = np.random.RandomState(seed)
        self.out_dtype = out_dtype or (torch.bfloat16 if self.cuda else torch.float32)
        N, H, W, C = self.raw_shape
        self.mean = torch.as_tensor(np.asarray(mean, dtype=np.float32)).to(self.device)
        if np.ndim(std_scale) > 0:                       # per-channel 1/(255·img_std) (ref proc_load_mpi.py:99)
            self.std_scale = torch.as_tensor(np.asarray(std_scale, dtype=np.float32)).to(self.device)
        else:
            self.std_scale = float(std_scale)
        pin = self.cuda
        self._on_close = on_close
        if host_buffers is not None:                     # ring owned by a loader process (shared memory, page-locked)
            assert len(host_buffers) == depth and all(tuple(t.shape) == self.raw_shape for t in host_buffers)
            self.host = list(host_buffers)
            self._ext_host = True
        else:
            self.host = [torch.empty(self.raw_shape, dtype=torch.uint8, pin_memory=pin) for _ in range(depth)]
            self._ext_host = False
        self.host_offs = [torch.empty((N, 2), dtype=torch.int32, pin_memory=pin) for _ in range(depth)]
        self.host_flip = [torch.empty((N,), dtype=torch.uint8, pin_memory=pin) for _ in range(depth)]
        self.resized_crop = resized_crop
        self.color_jitter = color_jitter
        if resized_crop is not None:
            self.rrc_rng = resized_crop_rng(resized_crop, rank)
        if color_jitter is not None:
            self.cj_rng = color_jitter_rng(color_jitter, rank)
            self.host_rec = [torch.empty((N, CJ_RECORD_FLOATS), dtype=torch.float32, pin_memory=pin) for _ in range(depth)]
        self.random_erasing = random_erasing
        if random_erasing is not None:
            self.re_rng = random_erasing_rng(random_erasing, rank)
            self.host_erase = [torch.empty((N, 4), dtype=torch.int32, pin_memory=pin) for _ in range(depth)]
        self.auto_augment = auto_augment
        if auto_augment is not None:
            self.aa_rng = auto_augment_rng(auto_augment, rank)
            self.aa_slots = aa_slots(auto_augment)
            self.aa_bilinear = aa_bilinear(auto_augment)
            self.host_aa = [torch.empty((N, self.aa_slots, AA_RECORD_FLOATS), dtype=torch.float32, pin_memory=pin)
                            for _ in range(depth)]
            self.aa_width = auto_augment["mixture_width"] if auto_augment["policy"] == "augmix" else 0
            if self.aa_width:
                self.host_aw = [torch.empty((N, 1 + self.aa_width), dtype=torch.float32, pin_memory=pin) for _ in range(depth)]
        boxed = resized_crop is not None or color_jitter is not None or auto_augment is not None
        if boxed:
            self.host_boxes = [torch.empty((N, 4), dtype=torch.int32, pin_memory=pin) for _ in range(depth)]
        if self.cuda:
            if boxed:
                self.dev_boxes = [torch.empty((N, 4), dtype=torch.int32, device=self.device) for _ in range(depth)]
            if color_jitter is not None:
                self.dev_rec = [torch.empty((N, CJ_RECORD_FLOATS), dtype=torch.float32, device=self.device) for _ in range(depth)]
                self.dev_mu = [torch.empty((N, 4), dtype=torch.float32, device=self.device) for _ in range(depth)]
            if auto_augment is not None:
                # the uint8 ping / pong crops and the point-op LUTs: used on the copy stream one batch at a time, so one set
                self.aa_ping = torch.empty((N,) + self.crop_hw + (3,), dtype=torch.uint8, device=self.device)
                self.aa_pong = torch.empty_like(self.aa_ping)
                self.aa_lut = torch.empty((N, 3, 256), dtype=torch.uint8, device=self.device)
                self.dev_aa = [torch.empty((N, self.aa_slots, AA_RECORD_FLOATS), dtype=torch.float32, device=self.device)
                               for _ in range(depth)]
                if self.aa_width:
                    # every chain starts from the crop in aa_ping, so the chains step through pairs of their own
                    self.aa_chains = torch.empty((self.aa_width, 2) + tuple(self.aa_ping.shape), dtype=torch.uint8, device=self.device)
                    self.dev_aw = [torch.empty((N, 1 + self.aa_width), dtype=torch.float32, device=self.device) for _ in range(depth)]
            if random_erasing is not None:
                self.dev_erase = [torch.empty((N, 4), dtype=torch.int32, device=self.device) for _ in range(depth)]
            self.stage = [torch.empty(self.raw_shape, dtype=torch.uint8, device=self.device) for _ in range(depth)]
            self.dev_offs = [torch.empty((N, 2), dtype=torch.int32, device=self.device) for _ in range(depth)]
            self.dev_flip = [torch.empty((N,), dtype=torch.uint8, device=self.device) for _ in range(depth)]
            self.copy_stream = torch.cuda.Stream(device=self.device)
            self.consumed = [None] * depth
        self.out = [torch.empty((N,) + self.crop_hw + (C,), dtype=self.out_dtype, device=self.device)
                    for _ in range(depth)]
        # slot s of this ring is slot s of self.out for a "val" batch: the same consumed[s] event guards both
        self.val_crops = val_crops
        self.val_out = None
        if val_crops > 1:
            self.val_out = [torch.empty((val_crops, N) + self.crop_hw + (C,), dtype=self.out_dtype, device=self.device)
                            for _ in range(depth)]
        self.h2d_bytes = int(np.prod(self.raw_shape)) + N * 9
        self._req = queue.Queue()
        self._done = queue.Queue()
        self._slot = 0
        self._last = None
        self.outstanding = 0
        self.threaded = threaded and self.cuda
        self._thread = None
        self._err = None
        if self.threaded:
            self._thread = threading.Thread(target=self._run, name="tmpi-loader", daemon=True)
            self._thread.start()

    # ------------------------------------------------------------------ producer
    def _produce(self, item, mode):
        s = self._slot
        self._slot = (s + 1) % self.depth
        N, H, W, C = self.raw_shape
        if self.cuda and self.consumed[s] is not None:
            self.consumed[s].synchronize()          # trainer finished reading slot s
        src = self.read_fn(item, self.host[s].numpy())          # may return its own pinned uint8 tensor (zero host copy)
        if not (isinstance(src, torch.Tensor) and src.dtype == torch.uint8 and tuple(src.shape) == self.raw_shape
                and (not self.cuda or src.is_pinned())):
            src = self.host[s]
        if self.cuda and self._ext_host and src is self.host[s]:
            # the ring slot is refilled by another process as soon as we request the next file: the DMA out of it must have
            # finished before this slot comes round again — recorded below, awaited at the top of the next _produce(s)
            pass
        aa = None
        if mode == "val" and self.val_crops > 1:
            # every view from the one staged copy; no draw, so self.rs and the training crops stay the same sequence
            if self.cuda:
                with torch.cuda.stream(self.copy_stream):
                    self.stage[s].copy_(src, non_blocking=True)
                    from ...ops import cuda_impl
                    cuda_impl.multi_crop_normalize(self.stage[s], self.mean, self.std_scale, self.crop_hw, self.val_crops,
                                                   self.out_dtype, out=self.val_out[s])
                ready = torch.cuda.Event()
                ready.record(self.copy_stream)
            else:
                self.val_out[s].copy_(ops.reference.multi_crop_normalize(src, self.mean, self.std_scale, self.crop_hw, self.val_crops))
                ready = None
            return LoadedBatch(self.val_out[s], s, ready, item, self.h2d_bytes)
        if mode == "train" and (self.resized_crop is not None or self.color_jitter is not None or self.auto_augment is not None):
            boxes, flips, records, aa, aw, nbytes = self._produce_boxed(s, src, mode)
        else:
            boxes = flips = records = aw = None
            nbytes = self.h2d_bytes
            offs, fl = draw_crops(N, (H, W), self.crop_hw, mode, self.rand_crop, self.batch_crop_mirror, self.rs)
            self.host_offs[s].numpy()[...] = offs
            self.host_flip[s].numpy()[...] = fl
            if self.cuda:
                with torch.cuda.stream(self.copy_stream):
                    self.stage[s].copy_(src, non_blocking=True)
                    self.dev_offs[s].copy_(self.host_offs[s], non_blocking=True)
                    self.dev_flip[s].copy_(self.host_flip[s], non_blocking=True)
                    from ...ops import cuda_impl
                    cuda_impl.crop_mirror_normalize(self.stage[s], self.mean, self.std_scale, self.crop_hw,
                                                    self.dev_offs[s], self.dev_flip[s], self.out_dtype,
                                                    out=self.out[s])
            else:
                x = ops.reference.crop_mirror_normalize(src, self.mean, self.std_scale, self.crop_hw,
                                                        self.host_offs[s], self.host_flip[s], self.out_dtype)
                self.out[s].copy_(x)
        erase = None
        if mode == "train" and self.random_erasing is not None:
            # the erase boxes come after whichever crop path ran, from their own generator, in output coordinates
            erase = draw_erase_boxes(N, self.crop_hw, self.random_erasing, self.re_rng)
            self.host_erase[s].numpy()[...] = erase
            nbytes += N * 16
            if self.cuda:
                with torch.cuda.stream(self.copy_stream):
                    self.dev_erase[s].copy_(self.host_erase[s], non_blocking=True)
                    from ...ops import cuda_impl
                    cuda_impl.random_erase(self.out[s], self.dev_erase[s])
            else:
                self.out[s].copy_(ops.reference.random_erase(self.out[s], self.host_erase[s]))
        ready = None
        if self.cuda:
            ready = torch.cuda.Event()
            ready.record(self.copy_stream)
        return LoadedBatch(self.out[s], s, ready, item, nbytes, boxes, flips, records, erase, aa, aw)

    def _produce_boxed(self, s, src, mode):
        """A "train" batch with ``resized_crop`` or ``color_jitter``: boxes (the random-resized-crop draw, or the fixed crops'
        offsets with the output's size) and flips drawn on the host, the 16-byte box record copied next to the flips, and the
        96-byte colour record with them under ``color_jitter``; then on the copy stream ``resized_crop_mirror_norm``, or
        ``crop_mean`` (only when the contrast strength is > 0, since otherwise K ≡ 0) and ``color_crop_mirror_norm`` (the
        references on the CPU).  Under ``auto_augment`` the op records (48 bytes per image and slot) travel with them and
        ``auto_augment_crop_normalize`` runs instead: the uint8 crop, per slot a LUT launch when a point op is drawn and an apply
        launch, then the normalisation; under "augmix" the weight records (4·(1 + width) bytes per image) travel too and the chains
        and the mix run between them.  Returns (boxes, flips, colour records or None, op records or None, AugMix weights or None,
        bytes copied)."""
        N, H, W, C = self.raw_shape
        if self.resized_crop is not None:
            boxes, flips = draw_resized_crops(N, (H, W), self.resized_crop["scale"], self.resized_crop["ratio"], self.rrc_rng)
        else:
            offs, flips = draw_crops(N, (H, W), self.crop_hw, mode, self.rand_crop, self.batch_crop_mirror, self.rs)
            boxes = np.concatenate([offs, np.tile(np.int32([self.crop_hw]), (N, 1))], 1)
        self.host_boxes[s].numpy()[...] = boxes
        self.host_flip[s].numpy()[...] = flips
        nbytes = int(np.prod(self.raw_shape)) + N * 17
        records = None
        if self.color_jitter is not None:
            records = color_jitter_records(N, self.color_jitter, self.cj_rng)[0]
            self.host_rec[s].numpy()[...] = records
            nbytes += N * 4 * CJ_RECORD_FLOATS
        aa = aw = None
        if self.auto_augment is not None:
            if self.aa_width:
                aa, aw, aa_ops, _ = augmix_records(N, self.auto_augment, self.aa_rng, self.crop_hw)
                self.host_aw[s].numpy()[...] = aw
                nbytes += aw.nbytes
            else:
                aa, aa_ops, _ = auto_augment_records(N, self.auto_augment, self.aa_rng, self.crop_hw)
            self.host_aa[s].numpy()[...] = aa
            nbytes += aa.nbytes
        if self.cuda:
            with torch.cuda.stream(self.copy_stream):
                self.stage[s].copy_(src, non_blocking=True)
                self.dev_boxes[s].copy_(self.host_boxes[s], non_blocking=True)
                self.dev_flip[s].copy_(self.host_flip[s], non_blocking=True)
                from ...ops import cuda_impl
                if aa is not None:
                    self.dev_aa[s].copy_(self.host_aa[s], non_blocking=True)
                    dw = None
                    if aw is not None:
                        dw = self.dev_aw[s]
                        dw.copy_(self.host_aw[s], non_blocking=True)
                    cuda_impl.auto_augment_crop_normalize(self.stage[s], self.mean, self.std_scale, self.crop_hw, self.dev_boxes[s],
                                                          self.dev_flip[s], self.dev_aa[s], aa_ops, self.out_dtype, out=self.out[s],
                                                          ping=self.aa_ping, pong=self.aa_pong, lut=self.aa_lut,
                                                          bilinear=self.aa_bilinear, weights=dw,
                                                          chains=self.aa_chains if dw is not None else None)
                elif records is None:
                    cuda_impl.resized_crop_mirror_normalize(self.stage[s], self.mean, self.std_scale, self.crop_hw, self.dev_boxes[s],
                                                            self.dev_flip[s], self.out_dtype, out=self.out[s])
                else:
                    self.dev_rec[s].copy_(self.host_rec[s], non_blocking=True)
                    mu = None
                    if self.color_jitter["contrast"] > 0:
                        mu = cuda_impl.crop_mean(self.stage[s], self.dev_boxes[s], self.crop_hw, out=self.dev_mu[s])
                    cuda_impl.color_crop_mirror_normalize(self.stage[s], self.mean, self.std_scale, self.crop_hw, self.dev_boxes[s],
                                                          self.dev_flip[s], self.dev_rec[s], mu, self.out_dtype, out=self.out[s])
        else:
            if aa is not None:
                x = ops.reference.auto_augment_crop_normalize(src, self.mean, self.std_scale, self.crop_hw, self.host_boxes[s],
                                                              self.host_flip[s], self.host_aa[s], self.out_dtype,
                                                              weights=self.host_aw[s] if aw is not None else None)
            elif records is None:
                x = ops.reference.resized_crop_mirror_normalize(src, self.mean, self.std_scale, self.crop_hw, self.host_boxes[s],
                                                                self.host_flip[s], self.out_dtype)
            else:
                x = ops.reference.color_crop_mirror_normalize(src, self.mean, self.std_scale, self.crop_hw, self.host_boxes[s],
                                                              self.host_flip[s], self.host_rec[s], self.out_dtype)
            self.out[s].copy_(x)
        return boxes, flips, records, aa, aw, nbytes

    def _run(self):
        if self.cuda:
            torch.cuda.set_device(self.device)
        while True:
            req = self._req.get()
            if req is None:
                break
            try:
                self._done.put(self._produce(*req))
            except Exception as e:  # surface in the trainer thread
                self._err = e
                self._done.put(None)
                break

    # ------------------------------------------------------------------ consumer API
    def set_mode(self, mode):
        self.mode = mode

    def request(self, item, mode=None):
        """Ask for ``item`` to be loaded (the reference's ``icomm.isend(filename, tag=40)``)."""
        req = (item, mode or self.mode)
        if self._last is not None:
            # the trainer has already enqueued every read of the batch it was handed last (the copy into its input buffer
            # happens at the start of its step): mark it consumed NOW, before the producer may pick that slot again
            self.release(self._last)
        self.outstanding += 1
        if self.threaded:
            self._req.put(req)
        else:
            self._done.put(self._produce(*req))

    def get(self):
        """Block until the oldest requested batch is in flight to the device, make the
        current stream wait for it, and hand it out (``icomm.recv('copy_finished', tag=55)``)."""
        if self._last is not None:
            self.release(self._last)
        b = self._done.get()
        self.outstanding -= 1
        if b is None:
            raise RuntimeError("loader thread failed: %r" % (self._err,))
        if self.cuda and b.ready is not None:
            torch.cuda.current_stream(self.device).wait_event(b.ready)
        self._last = b
        return b

    def release(self, b):
        """Mark the batch consumed (recorded on the trainer's stream)."""
        if self.cuda:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.device))
            self.consumed[b.slot] = ev
        if self._last is b:
            self._last = None

    def drain(self):
        """Consume look-ahead requests that will not be used (mode switch / epoch end)."""
        while self.outstanding > 0:
            self.get()
        if self._last is not None:
            self.release(self._last)

    def close(self):
        if self._thread is not None:
            self._req.put(None)
            self._thread.join(timeout=10)
            self._thread = None
        if self.cuda:
            torch.cuda.synchronize(self.device)
        if self._on_close is not None:
            self._on_close()
            self._on_close = None
