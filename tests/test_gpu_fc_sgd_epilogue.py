"""The momentum-SGD epilogue of the FC weight-gradient GEMM (``cuda_impl.gemm_sgd``) against its reference route, "GEMM into G
then ``sgd_flat``": the fused update must give the same bits."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _arena(O, I, seed):
    from theanompi_b200.parallel.arena import FlatArena
    g = torch.Generator().manual_seed(seed)
    w = torch.nn.Parameter(torch.randn(O, I, generator=g) * 0.05)
    w.pname = "W"
    a = FlatArena([w], device="cuda:0", weight_decay=5e-4)
    a.U[:O * I].copy_((torch.randn(O * I, generator=g) * 0.01).cuda())
    a.hyper[0] = 0.01
    return a, w


@pytest.mark.gpu
@pytest.mark.parametrize("O,I,B", [(4096, 9216, 128), (1000, 4096, 128), (16, 4096, 32), (264, 1032, 40), (264, 56, 40)])
@pytest.mark.parametrize("dtype", ["bf16", "tf32"])
@pytest.mark.parametrize("mu,nesterov", [(0.0, False), (0.9, False), (0.9, True)])
def test_fused_update_matches_gemm_then_sgd_flat(O, I, B, dtype, mu, nesterov):
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.utils.opt import FlatSGD
    adt = torch.bfloat16 if dtype == "bf16" else torch.float32
    g = torch.Generator().manual_seed(1)
    dy = torch.randn(B, O, generator=g).to(adt).cuda()
    x = torch.randn(B, I, generator=g).to(adt).cuda()
    ref, w_ref = _arena(O, I, 7)
    fus, w_fus = _arena(O, I, 7)
    # reference: the fp32 gradient GEMM into G, then the flat update over the tensor's blocks
    cuda_impl.gemm(dy, x, O, I, B, a_mn=True, b_mn=True, out=w_ref.gbuf, lda=O, ldb=I, ldc=I)
    cuda_impl.sgd_flat(ref, ref.G, 0.01, mu, nesterov, 1.0, 0, ref.numel)
    # fused
    sgd = FlatSGD(fus, mu, nesterov)
    w_fus.sgd_epilogue, w_fus.arena_group = sgd, fus.group_of[0]
    fus.G.fill_(float("nan"))
    cuda_impl.gemm_sgd(dy, x, w_fus, O, I, B, lda=O, ldb=I)
    torch.cuda.synchronize()
    n = O * I
    assert torch.equal(ref.W[:n], fus.W[:n])
    assert torch.equal(ref.U[:n], fus.U[:n])
    assert torch.equal(ref.H[:n], fus.H[:n])
    assert not torch.equal(ref.W[:n], w_ref.detach().new_zeros(n))


def test_armed_set_and_complement_cover_the_arena():
    """CPU: for AlexNet the armed weights are fc6.W, fc7.W and softmax.W, and armed ranges + complement tile the arena."""
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.parallel.arena import BLOCK
    from theanompi_b200.utils.opt import _fc_fusable, complement_ranges
    m = AlexNet(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=4, n_class=16,
                     data_kwargs=dict(n_train_files=1, n_val_files=1, synthetic=True)))
    a = m.arena
    armed = [i for i, p in enumerate(a.params) if _fc_fusable(p, 8)]
    # fc6.W, fc7.W, softmax.W
    assert [tuple(a.params[i].shape) for i in armed] == [(4096, 9216), (4096, 4096), (16, 4096)]
    assert a.params[armed[-1]] is m.output_layer.W.val
    cover = torch.zeros(a.numel, dtype=torch.int32)
    for i in armed:
        o = a.offsets[i]
        cover[o:o + -(-a.sizes[i] // BLOCK) * BLOCK] += 1
    for lo, hi in complement_ranges(a, armed):
        assert lo % BLOCK == 0 and hi % BLOCK == 0
        cover[lo:hi] += 1
    assert bool((cover == 1).all())


_TRAIN = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
from theanompi_b200.models import layers2
from theanompi_b200.models.alex_net import AlexNet
from theanompi_b200.ops import cuda_impl
from theanompi_b200.utils.recorder import Recorder

def run(graph, armed, nan_g):
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); cuda_impl._STEP.clear()
    m = AlexNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=32, file_batch_size=32, n_class=16, cuda_graph=graph,
                     data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True)))
    m.monitor_grad = not armed          # gradient monitoring reads G, so it keeps the GEMM-into-G route
    m.compile_iter_fns("avg")
    ps = [p for p in m.arena.params if getattr(p, "sgd_epilogue", None) is not None]
    assert len(ps) == (3 if armed else 0), len(ps)
    rec = Recorder(None, 10 ** 6, "AlexNet", False, device="cuda:0")
    losses = []
    for i in range(5):
        if nan_g:
            for p in ps:
                p.gbuf.fill_(float("nan"))
        m.train_iter(i, rec)
        losses.append(float(rec.train_info["cost"][-1]))
    torch.cuda.synchronize()
    if armed:
        try:
            m.grad_norms()
            raise AssertionError("grad_norms() read G of armed weights")
        except RuntimeError:
            pass
    out = (losses, m.arena.W.clone(), m.arena.U.clone())
    m.cleanup()
    return out

for graph in (False, True):
    l0, w0, u0 = run(graph, False, False)
    for nan_g in (False, True):
        l1, w1, u1 = run(graph, True, nan_g)
        assert l0 == l1, (graph, nan_g, l0, l1)
        bad = (w0 != w1).nonzero().flatten()
        assert bad.numel() == 0 and torch.equal(u0, u1), (graph, nan_g, bad.numel(), bad[:4].tolist())
print("ok")
"""


@pytest.mark.gpu
def test_alexnet_armed_matches_unarmed_bitwise(tmp_path):
    """AlexNet (batch 32, 16 classes), eager and CUDA graph, 5 steps: the armed model computes exactly what the GEMM-into-G
    route computes, also with NaN in the armed weights' G (nothing reads it), and the gradient monitor refuses to read G of
    armed weights.  Deterministic kernels, so it runs in its own process."""
    env = dict(os.environ, TMPI_DETERMINISTIC="1")
    r = subprocess.run([sys.executable, "-c", _TRAIN, ROOT], env=env, cwd=str(tmp_path), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-4000:]
