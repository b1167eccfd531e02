"""CPU: the checks GraphedTrainStep makes before it touches a GPU, make_optimizer's fused switch, and fused.weights_updated."""
import pytest
import torch
import torch.nn as nn


def _model():
    return nn.Sequential(nn.Conv2d(6, 8, 1), nn.LayerNorm(1))


def _example():
    return torch.zeros(2, 3, 4, 4), torch.zeros(2, 3, 4, 4), torch.zeros(2, 4, 4, dtype=torch.long)


def test_make_optimizer_defaults_unchanged_and_fused_switch():
    from sigma_b200 import train_util
    m = _model()
    opt = train_util.make_optimizer(m)
    assert all(g["fused"] is None and g["capturable"] is False for g in opt.param_groups)
    assert not getattr(opt, "_step_supports_amp_scaling", False)
    assert [len(g["params"]) for g in opt.param_groups] == [len(g["params"]) for g in train_util.group_weight(m, 6e-5)]


def test_rejects_uncapturable_optimizer():
    from sigma_b200 import train_util
    m = _model()
    with pytest.raises(ValueError, match="capturable=True or fused=True"):
        train_util.GraphedTrainStep(m, train_util.make_optimizer(m), _example())


def test_rejects_scaler_without_device_side_skip():
    from sigma_b200 import train_util
    m = _model()
    scaler = torch.amp.GradScaler("cpu")
    assert scaler.is_enabled()
    with pytest.raises(ValueError, match="fused=True"):
        train_util.GraphedTrainStep(m, train_util.make_optimizer(m, capturable=True), _example(), scaler=scaler)


def test_rejects_host_example_and_no_warmup():
    from sigma_b200 import train_util
    m = _model()
    opt = train_util.make_optimizer(m, capturable=True)
    with pytest.raises(ValueError, match="CUDA tensors"):
        train_util.GraphedTrainStep(m, opt, _example())
    with pytest.raises(ValueError, match="CUDA tensors"):
        train_util.GraphedTrainStep(m, opt, _example()[:2])
    with pytest.raises(ValueError, match="warmup"):
        train_util.GraphedTrainStep(m, opt, _example(), warmup=0)


def test_rejects_ddp(tmp_path):
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel
    from sigma_b200 import train_util
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'pg'}", rank=0, world_size=1)
    try:
        ddp = DistributedDataParallel(_model())
        with pytest.raises(ValueError, match="DistributedDataParallel"):
            train_util.GraphedTrainStep(ddp, train_util.make_optimizer(ddp, capturable=True), _example())
    finally:
        dist.destroy_process_group()


def test_weights_updated_bumps_every_version_once():
    from sigma_b200 import fused
    m = _model()
    ps = list(m.parameters())
    v0 = [p._version for p in ps]
    fused.weights_updated(ps)
    assert [p._version for p in ps] == [v + 1 for v in v0]
    built = []
    key = lambda: tuple((p._version, p.data_ptr()) for p in ps)   # noqa: E731  (the key fused._ssm_params uses)
    fused._cache(m, "t", key(), lambda: built.append(1))
    fused._cache(m, "t", key(), lambda: built.append(1))
    fused.weights_updated(ps[:1])
    fused._cache(m, "t", key(), lambda: built.append(1))
    assert len(built) == 2
