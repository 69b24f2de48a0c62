"""CUDA-graph capture of a model step while unreachable models are waiting for the garbage collector: no automatic collection runs
inside the capture (finalising a dead model's CUDA graph there makes a call a capturing thread must not make, which invalidates the
capture), and the collector is on again after it."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WRN = dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=16, file_batch_size=16, depth=10, widen=1, cuda_graph=True,
           data_kwargs=dict(n_synthetic=64, synthetic=True))


def _wrn():
    from theanompi_b200.models import layers2
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)
    m = Wide_ResNet(dict(WRN))
    m.compile_iter_fns("avg")
    return m


def _train(m, steps):
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
    for i in range(steps):
        m.train_iter(i, rec)
    torch.cuda.synchronize()


def test_capture_survives_a_dead_captured_model_and_no_collection_runs_inside_it():
    holder = [_wrn()]
    _train(holder[0], 4)
    assert holder[0].captured_steps() == {"step"}
    holder[0]._cycle = holder[0]                  # unreachable once dropped from holder: only the collector frees it

    m = _wrn()
    body, seen = m._step_body, []

    def step_body(kind="step"):
        seen.append(gc.isenabled())
        if len(seen) == 3:                        # the capture: the dead model becomes garbage while it runs
            holder.clear()
        return body(kind)
    m._step_body = step_body
    threshold = gc.get_threshold()
    gc.set_threshold(1, 1, 1)                     # an automatic collection on nearly every allocation
    try:
        _train(m, 5)
    finally:
        gc.set_threshold(*threshold)
    assert seen[:2] == [True, True] and seen[2] is False, seen    # the two eager warm-ups, then the capture
    assert len(seen) == 3 and gc.isenabled()      # later steps replay the graph
    assert m.captured_steps() == {"step"}
    gc.collect()
