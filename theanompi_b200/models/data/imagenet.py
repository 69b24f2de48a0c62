"""ImageNet batch-file dataset (ref ``theanompi/models/data/imagenet.py``).

Same API: ``batch_data`` (``:109-148``), ``extend_data`` (``:150-164``),
``shuffle_data(mode, common_seed)`` — the SAME permutation on every rank
(``:167-199``), ``shard_data`` = ``list[rank::size]`` (``:205-222``), ``spawn_load`` /
``para_load_init`` / ``para_load_close`` (``:226-321``).

Storage: one ``.npy`` file per 128-image batch, uint8 NHWC ``[128,256,256,3]``
(the reference used hickle ``.hkl`` in c01b layout; ``.hkl`` files are read too when the ``hickle`` package is
importable — it is not part of this image — and transposed to NHWC).  When
the directory does not exist the dataset is **synthetic**: file names are
``synthetic://<split>/<index>`` and ``read`` fills the pinned buffer from a small
pool of pre-generated random batches (there is no network / dataset in the build
and bench environment); labels are a fixed function of the index.
"""
from __future__ import annotations

import glob
import os

import numpy as np

from .utils import extend_data as _extend

dir_head = os.environ.get("TMPI_IMAGENET_DIR", "./prepdata_1000cat_128b/")
label_folder = "/labels/"
mean_file = "/misc/img_mean.npy"
train_folder = "/train_npy_128b/"
val_folder = "/val_npy_128b/"
para_load = True
debug = False


class ImageNet_data(object):
    def __init__(self, verbose=False, synthetic=None, n_train_files=40, n_val_files=8,
                 file_batch_size=128, size_hw=256, pool=4, seed=0, n_class=1000):
        self.data_path = dir_head
        self.channels = 3
        self.width = self.height = size_hw
        self.n_class = n_class
        self.verbose = verbose
        self.batched = False
        self.extended = False
        self.para_load = para_load
        self.file_batch_size = file_batch_size
        self.loader = None
        if synthetic is None:
            synthetic = not os.path.isdir(self.data_path + train_folder)
        self.synthetic = synthetic
        self._pool_n = pool
        self._pool = None
        self._seed = seed
        self.n_syn = (n_train_files, n_val_files)
        self.get_data(file_batch_size)

    # ------------------------------------------------------------------ raw data
    def get_data(self, file_batch_size=128):
        if self.synthetic:
            ntr, nva = self.n_syn
            train_filenames = ["synthetic://train/%06d" % i for i in range(ntr)]
            val_filenames = ["synthetic://val/%06d" % i for i in range(nva)]
            rs = np.random.RandomState(self._seed + 17)
            train_labels = rs.randint(0, self.n_class, ntr * file_batch_size).astype(np.int64)
            val_labels = rs.randint(0, self.n_class, nva * file_batch_size).astype(np.int64)
            img_mean = np.full((self.height, self.width, self.channels), 127.5, dtype=np.float32)
        else:
            train_filenames = sorted(glob.glob(self.data_path + train_folder + "/*.npy") +
                                     glob.glob(self.data_path + train_folder + "/*.hkl"))
            val_filenames = sorted(glob.glob(self.data_path + val_folder + "/*.npy") +
                                   glob.glob(self.data_path + val_folder + "/*.hkl"))
            if debug:
                train_filenames, val_filenames = train_filenames[:40], val_filenames[:20]
            train_labels = np.load(self.data_path + label_folder + "train_labels.npy")
            val_labels = np.load(self.data_path + label_folder + "val_labels.npy")
            img_mean = np.load(self.data_path + mean_file).astype(np.float32)
            if img_mean.shape[0] == 3:                      # reference stores c01
                img_mean = np.transpose(img_mean, (1, 2, 0))
        img_std = np.array([0.229, 0.224, 0.225], dtype=np.float32)
        self.rawdata = [train_filenames, train_labels, val_filenames, val_labels, img_mean, img_std]

    def read(self, filename, out):
        """Fill ``out`` (uint8 NHWC numpy view of a pinned buffer) with one file batch."""
        if filename.startswith("synthetic://"):
            import torch
            if self._pool is None:
                rs = np.random.RandomState(self._seed)
                pin = torch.cuda.is_available()
                self._pool = []
                for _ in range(self._pool_n):                      # synthetic "files" live in pinned memory
                    t = torch.empty(tuple(out.shape), dtype=torch.uint8, pin_memory=pin)
                    t.numpy()[...] = rs.randint(0, 256, out.shape, dtype=np.uint8)
                    self._pool.append(t)
            idx = int(filename.rsplit("/", 1)[1])
            src = self._pool[idx % self._pool_n]
            if getattr(self, "zero_copy", True):
                return src                                          # the loader DMAs straight from this buffer
            np.copyto(out, src.numpy())
        elif filename.endswith(".hkl"):
            try:
                import hickle
            except ImportError as e:
                raise RuntimeError("%s: reading the reference's .hkl batches needs the hickle package; convert them to .npy "
                                   "(uint8 NHWC) instead" % filename) from e
            arr = np.asarray(hickle.load(filename))
            if arr.ndim == 4 and arr.shape[0] == self.channels:        # reference layout c01b → b01c
                arr = np.transpose(arr, (3, 1, 2, 0))
            np.copyto(out, arr.astype(np.uint8, copy=False))
        else:
            from .utils import parallel_copyto
            arr = np.load(filename, mmap_mode="r")
            parallel_copyto(out, arr)

    # ------------------------------------------------------------------ batching / sharding
    def batch_data(self, file_batch_size):
        if self.batched:
            return
        self.n_batch_train = len(self.rawdata[0])
        self.n_batch_val = len(self.rawdata[2])
        if self.verbose:
            print("train on %d files" % self.n_batch_train)
            print("val on %d files" % self.n_batch_val)
        self.train_img, self.val_img = list(self.rawdata[0]), list(self.rawdata[2])
        self.train_labels = [self.rawdata[1][i * file_batch_size:(i + 1) * file_batch_size]
                             for i in range(self.n_batch_train)]
        self.val_labels = [self.rawdata[3][i * file_batch_size:(i + 1) * file_batch_size]
                           for i in range(self.n_batch_val)]
        self.batched = True

    def extend_data(self, rank, size):
        if self.extended:
            return
        if not self.batched:
            raise RuntimeError("extend_data needs to be after batch_data")
        self.train_img_ext, self.train_labels_ext = _extend(rank, size, self.train_img, self.train_labels, self.verbose)
        self.val_img_ext, self.val_labels_ext = _extend(rank, size, self.val_img, self.val_labels, self.verbose)
        self.n_batch_train = len(self.train_img_ext)
        self.n_batch_val = len(self.val_img_ext)
        self.extended = True

    def shuffle_data(self, mode, common_seed=1234):
        if not self.extended:
            raise RuntimeError("shuffle_data needs to be after extend_data")
        if mode == "train":
            rs = np.random.RandomState(common_seed)
            self.n_batch_train = len(self.train_img_ext)
            indices = rs.permutation(self.n_batch_train)
            self.train_img_shuffle = [self.train_img_ext[i] for i in indices]
            self.train_labels_shuffle = [self.train_labels_ext[i] for i in indices]
            if self.verbose:
                print("training data shuffled", indices[:8], "...")
        else:
            self.val_img_shuffle = self.val_img_ext
            self.val_labels_shuffle = self.val_labels_ext

    def shard_data(self, mode, rank, size):
        if mode == "train":
            self.train_img_shard = self.train_img_shuffle[rank::size]
            self.train_labels_shard = self.train_labels_shuffle[rank::size]
            self.n_batch_train = len(self.train_img_shard)
            if self.verbose:
                print("training data sharded", self.n_batch_train)
        else:
            self.val_img_shard = self.val_img_shuffle[rank::size]
            self.val_labels_shard = self.val_labels_shuffle[rank::size]
            self.n_batch_val = len(self.val_img_shard)
            if self.verbose:
                print("validation data sharded", self.n_batch_val)

    def load_batch(self, item, mode, model):
        """Serial (no loader) path of the reference (``alex_net.py:420-438``): read, normalise,
        crop/mirror on the host, return an NHWC float tensor.  With ``model.resized_crop`` a "train" batch is the random-resized
        crop of :meth:`para_load_init`'s loader, drawn from this object's generator keyed by (seed, ``model.rank``).  With
        ``model.color_jitter`` a "train" batch also gets the loader's colour maps, drawn from a generator keyed by (seed, rank, 1),
        on the same boxes or fixed crops as without it.  With ``model.random_erasing`` a "train" batch, whichever crop made it, then
        gets the loader's erase boxes, drawn from a generator keyed by (seed, rank, 3), set to 0.  With ``model.auto_augment`` a
        "train" batch gets the loader's op records (and, for "augmix", its mixing weights), drawn from a generator keyed by (seed,
        rank, 2), on the same boxes or fixed crops.  With ``model.val_crops`` = V > 1 a "val" batch is the view-major [V, N, ...] of ``reference.multi_crop_normalize``."""
        import torch
        from ... import ops
        from .utils import color_jitter_records, color_jitter_rng, crop_and_mirror, draw_crops
        raw = np.empty((self.file_batch_size, self.height, self.width, self.channels), dtype=np.uint8)
        src = self.read(item, raw)
        if src is not None:
            raw = src.numpy()
        rrc = getattr(model, "resized_crop", None)
        cj = getattr(model, "color_jitter", None) if mode == "train" else None
        aa = getattr(model, "auto_augment", None) if mode == "train" else None
        n = raw.shape[0]
        mean, cs = torch.from_numpy(self.rawdata[4]), torch.from_numpy(1.0 / 255.0 / self.rawdata[5])
        n_views = getattr(model, "val_crops", 1) if mode == "val" else 1
        if n_views > 1:
            t = ops.reference.multi_crop_normalize(torch.from_numpy(raw), mean, cs, (model.input_height, model.input_width), n_views)
            return t.pin_memory().to(model.device, non_blocking=True) if model.cuda else t
        if rrc is not None and mode == "train":
            from .utils import draw_resized_crops, resized_crop_rng
            if getattr(self, "_rrc_rng", None) is None:
                self._rrc_rng = resized_crop_rng(rrc, model.rank)
            out_hw = (model.input_height, model.input_width)
            boxes, flips = draw_resized_crops(n, (self.height, self.width), rrc["scale"], rrc["ratio"], self._rrc_rng)
            if cj is None and aa is None:
                t = ops.reference.resized_crop_mirror_normalize(torch.from_numpy(raw), mean, cs, out_hw, boxes, flips)
        elif cj is not None or aa is not None:
            # the same RandomState draw as crop_and_mirror below, so the key changes no crop
            out_hw = (model.input_width, model.input_width)
            offs, flips = draw_crops(n, (self.height, self.width), out_hw, mode, model.rand_crop, model.batch_crop_mirror)
            boxes = np.concatenate([offs, np.tile(np.int32([out_hw]), (n, 1))], 1)
        else:
            arr = (raw.astype(np.float32) - self.rawdata[4]) / 255.0 / self.rawdata[5]
            arr = crop_and_mirror(arr, mode, model.rand_crop, model.batch_crop_mirror, model.input_width)
            t = torch.from_numpy(arr)
        if cj is not None:
            if getattr(self, "_cj_rng", None) is None:
                self._cj_rng = color_jitter_rng(cj, model.rank)
            records = color_jitter_records(n, cj, self._cj_rng)[0]
            t = ops.reference.color_crop_mirror_normalize(torch.from_numpy(raw), mean, cs, out_hw, boxes, flips, records)
        if aa is not None:
            from .utils import augmix_records, auto_augment_records, auto_augment_rng
            if getattr(self, "_aa_rng", None) is None:
                self._aa_rng = auto_augment_rng(aa, model.rank)
            weights = None
            if aa["policy"] == "augmix":
                records, weights = augmix_records(n, aa, self._aa_rng, out_hw)[:2]
            else:
                records = auto_augment_records(n, aa, self._aa_rng, out_hw)[0]
            t = ops.reference.auto_augment_crop_normalize(torch.from_numpy(raw), mean, cs, out_hw, boxes, flips, records,
                                                          weights=weights)
        re_cfg = getattr(model, "random_erasing", None) if mode == "train" else None
        if re_cfg is not None:
            from .utils import draw_erase_boxes, random_erasing_rng
            if getattr(self, "_re_rng", None) is None:
                self._re_rng = random_erasing_rng(re_cfg, model.rank)
            t = ops.reference.random_erase(t, draw_erase_boxes(n, tuple(t.shape[1:3]), re_cfg, self._re_rng))
        if model.cuda:
            t = t.pin_memory().to(model.device, non_blocking=True)
        return t

    # ------------------------------------------------------------------ parallel loading
    def spawn_load(self):
        """The reference spawns an MPI child here (``:226-267``); here the loader (thread + copy stream, or with
        ``TMPI_LOADER=process`` a child process filling a page-locked shared-memory ring) is created in
        :meth:`para_load_init`, once the input geometry is known."""
        return None

    def para_load_init(self, device, input_width, input_height, rand_crop, batch_crop_mirror,
                       out_dtype=None, depth=2, mode=None, resized_crop=None, rank=0, color_jitter=None, random_erasing=None,
                       auto_augment=None, val_crops=1):
        """``mode='thread'`` (default): loader thread + pinned ring in this process.  ``mode='process'`` (or
        ``TMPI_LOADER=process``): a separate loader process fills a page-locked shared-memory ring (see ``proc_loader.py``) —
        the reference's ``proc_load_mpi.py`` child, minus its second CUDA context.  ``resized_crop`` (a validated
        ``config['random_resized_crop']``), ``color_jitter`` (a validated ``config['color_jitter']``), ``random_erasing`` (a
        validated ``config['random_erasing']``) and ``rank`` go to the :class:`ParaLoader`, which draws the boxes, the colour maps
        and the erase boxes in this process.  ``val_crops`` > 1 makes it cut that many views of every "val" batch, also in this
        process."""
        from .loader import ParaLoader
        raw_shape = (self.file_batch_size, self.height, self.width, self.channels)
        mode = mode or os.environ.get("TMPI_LOADER", "thread")
        kw = dict(mean=self.rawdata[4], std_scale=1.0 / 255.0 / self.rawdata[5], out_dtype=out_dtype, depth=depth,
                  rand_crop=rand_crop, batch_crop_mirror=batch_crop_mirror, resized_crop=resized_crop, rank=rank,
                  color_jitter=color_jitter, random_erasing=random_erasing, auto_augment=auto_augment,
                  val_crops=val_crops)
        if mode == "process":
            from .proc_loader import ProcReader
            self.proc_reader = ProcReader(raw_shape, depth=depth, seed=self._seed)
            self.loader = ParaLoader(self.proc_reader.read, device, raw_shape, (input_height, input_width),
                                     host_buffers=self.proc_reader.tensors, on_close=self.proc_reader.close, **kw)
        else:
            self.loader = ParaLoader(self.read, device, raw_shape, (input_height, input_width), **kw)
        return self.loader

    def para_load_close(self):
        if self.loader is not None:
            self.loader.close()
            self.loader = None
