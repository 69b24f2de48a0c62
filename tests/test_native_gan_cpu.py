"""The native GAN models (NativeWGAN, NativeLSGAN, CIFAR-10 NativeLSGAN) on the CPU reference path: direct steps, and world
size 2 over gloo through the BSP exchanger and the public Rule API."""
import math
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZOO = "theanompi_b200.models.lasagne_model_zoo."
MODELS = [(ZOO + "wgan", "NativeWGAN", dict(critic_runs=2, data_kwargs=dict(n_synthetic=128))),
          (ZOO + "lsgan", "NativeLSGAN", dict(data_kwargs=dict(n_synthetic=128))),
          (ZOO + "lsgan_cifar10", "NativeLSGAN", dict(data_kwargs=dict(n_synthetic=128, synthetic=True)))]


@pytest.mark.parametrize("modelfile,modelclass,cfg", MODELS)
def test_native_gan_two_steps(modelfile, modelclass, cfg, tmp_path):
    import importlib
    from theanompi_b200.utils.recorder import Recorder
    m = getattr(importlib.import_module(modelfile), modelclass)(dict(verbose=False, rank=0, size=1, device="cpu", **cfg))
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, modelclass, False, device="cpu")
    w0, g0 = m.arena.W.clone(), m.gen_arena.W.clone()
    c = 0
    for _ in range(2):
        c = m.train_iter(c, rec)
    assert c == 2 * cfg.get("critic_runs", 1)                       # train_iter returns the advanced count
    m.val_iter(c, rec)
    assert all(math.isfinite(float(v)) for v in rec.train_info["cost"] + rec.train_info["error"] + rec.val_info["cost"])
    assert not torch.equal(w0, m.arena.W) and not torch.equal(g0, m.gen_arena.W)
    assert [p.data_ptr() for p in m.params] == [p.data_ptr() for p in m.critic_params]     # exchanged params = critic only
    if m.loss_kind == "wgan":
        assert float(m.arena.W.abs().max()) <= 0.01 + 1e-9
    C = m.image_ch                                                  # padded image channels keep zero weights
    assert torch.all(m.critic_params[0][..., C:] == 0) and torch.all(m.generator_params[12][..., C:] == 0)
    m.print_info(rec, verbose=False)
    m.save(str(tmp_path))
    m2 = type(m)(dict(verbose=False, rank=0, size=1, device="cpu", **cfg))
    m2.load(str(tmp_path), m.epoch)
    assert torch.equal(m2.arena.W, m.arena.W) and torch.equal(m2.gen_arena.W, m.gen_arena.W)


def test_native_gan_bsp_world2():
    import test_distributed_cpu as td                     # shares its port counter
    td._PORT[0] += 1
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(td._PORT[0]),
                   OMP_NUM_THREADS="2", PYTHONPATH=ROOT)
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "mp_gan_checks.py"), "native_gan_bsp"], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=300)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d failed:\n%s" % (r, o[-3000:])


def test_native_wgan_through_bsp_rule(tmp_path, monkeypatch):
    import theanompi_b200 as tm
    monkeypatch.chdir(tmp_path)
    tm.BSP.sync_type, tm.BSP.exch_strategy = "avg", "ar"
    rule = tm.BSP()
    rule.model_config = dict(n_epochs=1, epochsize=2, critic_runs=2, max_batches=2, printFreq=1, data_kwargs=dict(n_synthetic=128))
    rule.env["OMP_NUM_THREADS"] = "2"
    rule.init(devices=["cpu0", "cpu1"], modelfile=ZOO + "wgan", modelclass="NativeWGAN")
    try:
        rc = rule.proc.wait(timeout=300)
    except subprocess.TimeoutExpired:
        rule.proc.kill()
        raise
    assert rc == 0
    assert os.path.exists(tmp_path / "snapshots" / "ckpt_0.pt")
