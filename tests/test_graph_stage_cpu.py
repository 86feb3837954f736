"""CPU-only: the cuda_graph keyword and the --cuda-graph flags, the refusals that come before any work, and the
BatchNorm buffer save / restore that brackets the capture's warm-up."""
import importlib.util
import os

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(rel):
    spec = importlib.util.spec_from_file_location(os.path.basename(rel)[:-3], os.path.join(ROOT, "benchmarks", rel))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


@pytest.mark.parametrize("rel", ["spatial_parallelism/benchmark_sp.py",
                                 "gems_master_with_spatial_parallelism/benchmark_gems_master_with_sp.py"])
def test_training_scripts_parse_cuda_graph(rel):
    p = _load(rel).get_parser()
    a = p.parse_args(["--cuda-graph", "--recompute", "--dtype", "bf16-amp", "--deterministic"])
    assert a.cuda_graph and a.recompute and a.deterministic and a.dtype == "bf16-amp"
    assert not p.parse_args([]).cuda_graph


@pytest.mark.parametrize("trainer", ["train_model", "train_model_spatial", "train_model_master",
                                     "train_spatial_model_master"])
def test_trainers_take_cuda_graph_keyword(trainer):
    import inspect

    from mpi4dl_b200.torchgems import gems_master, mp_pipeline, train_spatial, train_spatial_master
    cls = {"train_model": mp_pipeline.train_model, "train_model_spatial": train_spatial.train_model_spatial,
           "train_model_master": gems_master.train_model_master,
           "train_spatial_model_master": train_spatial_master.train_spatial_model_master}[trainer]
    par = inspect.signature(cls.__init__).parameters["cuda_graph"]
    assert par.kind == par.KEYWORD_ONLY and par.default is False


def _stage(parts):
    from mpi4dl_b200.torchgems import spatial
    return nn.Sequential(spatial.conv_spatial(0, 1, parts, 3, 8, 3, padding=1), nn.BatchNorm2d(8), nn.ReLU())


def _gen(model):
    from mpi4dl_b200.torchgems.mp_pipeline import model_generator
    g = model_generator(model=model, split_size=1, input_size=(1, 3, 16, 16), shape_list=[(1, 8, 16, 16)])
    g.models = model
    return g


def test_cuda_graph_without_cuda_raises_before_any_work(monkeypatch):
    from mpi4dl_b200.torchgems import graphs
    from mpi4dl_b200.torchgems.mp_pipeline import train_model
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(graphs.GraphCaptureError, match="needs a CUDA device"):
        train_model(_gen(_stage(1)), 0, 1, 1, cuda_graph=True)
    train_model(_gen(_stage(1)), 0, 1, 1)                  # off: nothing changes


def test_cuda_graph_with_dist_transport_raises_before_any_work(monkeypatch):
    from mpi4dl_b200.torchgems import graphs, halo_transport
    from mpi4dl_b200.torchgems.mp_pipeline import train_model
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setenv("SPCONV_HALO_TRANSPORT", "dist")
    monkeypatch.setattr(halo_transport, "_transport", None)
    with pytest.raises(graphs.GraphCaptureError, match="DistTransport"):
        train_model(_gen(_stage(4)), 0, 1, 1, cuda_graph=True)
    assert halo_transport._transport is None               # the check itself set up no transport
    graphs.check_graphable(_stage(1))                      # a stage without neighbours exchanges nothing


def test_batchnorm_buffers_restored_around_warmup():
    from mpi4dl_b200.torchgems.recompute import restore_batchnorm_buffers, save_batchnorm_buffers
    torch.manual_seed(0)
    m = nn.Sequential(nn.Conv2d(3, 4, 3), nn.BatchNorm2d(4), nn.Sequential(nn.BatchNorm2d(4, momentum=None)),
                      nn.BatchNorm2d(4, track_running_stats=False)).train()
    before = [b.clone() for b in m.buffers()]
    saved = save_batchnorm_buffers(m)
    assert len(saved) == 2
    for _ in range(2):                                     # warm-up forwards move every running buffer
        m(torch.randn(2, 3, 8, 8)).sum().backward()
    assert not all(torch.equal(a, b) for a, b in zip(before, m.buffers()))
    restore_batchnorm_buffers(saved)
    assert all(torch.equal(a, b) for a, b in zip(before, m.buffers()))
    ref = nn.Sequential(nn.Conv2d(3, 4, 3), nn.BatchNorm2d(4)).train()
    ref.load_state_dict({k: v for k, v in m.state_dict().items() if k.split(".")[0] in ("0", "1")})
    x = torch.randn(2, 3, 8, 8)
    m(x)
    ref(x)
    assert torch.equal(m[1].running_mean, ref[1].running_mean) and int(m[1].num_batches_tracked) == 1
