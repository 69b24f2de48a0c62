"""The loader handshake when train_iter / val_iter start a new pass over the files without reset_iter: every step holds the batch of
the file it asked for, next to that file's labels, with one look-ahead request in flight."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def test_a_new_pass_consumes_the_last_look_ahead():
    from theanompi_b200.models import layers2
    from theanompi_b200.models.alex_net import AlexNet
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear()
    m = AlexNet(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=4, n_class=8,
                     data_kwargs=dict(n_train_files=4, n_val_files=2, synthetic=True)))
    ld = m.data.loader
    try:
        for mode, img, lab, seq in (("train", m.data.train_img_shard, m.data.train_labels_shard, [0, 1, 2, 3, 0, 1, 2, 3, 0]),
                                    ("val", m.data.val_img_shard, m.data.val_labels_shard, [0, 1, 0, 1, 0])):
            m.reset_iter(mode)
            for idx in seq:
                m._load_file_batch(mode, idx, img, lab, len(img))
                assert ld._last.item == img[idx], (mode, idx)
                assert ld.outstanding == 1, (mode, idx)
                assert np.array_equal(m.shared_y[:4].numpy(), np.asarray(lab[idx])), (mode, idx)
    finally:
        m.cleanup()
