"""Host logic of checkpoint save / resume: when to save (against the reference's check_progress), where, the
fingerprint check, and the file layout written through a temporary directory."""
import os

import pytest
import torch

from rlinf_b200 import checkpoint as ckpt
from rlinf_b200.config import Cfg
from rlinf_b200.runner import check_save_config, should_evaluate, should_save


def test_should_save_matches_reference_check_progress(golden):
    table = golden("ckpt")["check_progress"]
    assert table[:, 4].sum() > 0 and table[:, 6].sum() > 0
    for step, max_steps, val, save, asserts, run_val, save_model in table.tolist():
        if asserts:
            with pytest.raises(ValueError, match="divisible"):
                should_save(step, max_steps, val, save)
            continue
        assert should_save(step, max_steps, val, save) == bool(save_model), (step, max_steps, val, save)
        assert should_evaluate(step, max_steps, val) == bool(run_val), (step, max_steps, val)


def _cfg(runner):
    return Cfg({"runner": runner})


def test_check_save_config():
    logger = {"log_path": "/logs", "experiment_name": "exp"}
    assert check_save_config(_cfg({}), 0) == 0
    assert check_save_config(_cfg({"save_interval": -1}), 2) == -1
    assert check_save_config(_cfg({"save_interval": 4, "logger": logger}), 2) == 4
    with pytest.raises(ValueError, match="divisible"):
        check_save_config(_cfg({"save_interval": 3, "logger": logger}), 2)
    with pytest.raises(ValueError, match="experiment_name"):
        check_save_config(_cfg({"save_interval": 1, "logger": {"log_path": "/logs"}}), 0)
    with pytest.raises(ValueError, match="log_path"):
        check_save_config(_cfg({"save_interval": 1}), 0)


def test_directory_naming_and_step_parsing():
    r = Cfg({"logger": {"log_path": "/logs", "experiment_name": "exp"}})
    d = ckpt.checkpoint_dir(r, 12)
    assert d == os.path.join("/logs", "exp", "checkpoints", "global_step_12")
    assert ckpt.step_from_path(d) == 12
    assert ckpt.step_from_path(d + os.sep) == 12
    assert ckpt.step_from_path("/a/global_step_3/b/global_step_40") == 40
    assert ckpt.rank_dir(d, 1) == os.path.join(d, "rank_1")
    with pytest.raises(ValueError, match="global_step_"):
        ckpt.step_from_path("/logs/exp/checkpoints/latest")


def _fp(**over):
    fp = {"obs_dim": 128, "action_dim": 8, "num_action_chunks": 1, "value_dim": 1, "world_size": 1,
          "total_num_envs": 4096, "max_steps_per_rollout_epoch": 512, "rollout_epoch": 1,
          "eval_total_num_envs": 0}
    fp.update(over)
    return fp


@pytest.mark.parametrize("field", ckpt.FINGERPRINT_FIELDS)
def test_fingerprint_mismatch_names_the_field(field):
    ckpt.check_fingerprint(_fp(), _fp())
    with pytest.raises(ValueError, match=field):
        ckpt.check_fingerprint(_fp(**{field: 2 * _fp()[field] + 1}), _fp())


def test_write_read_layout_and_replace(tmp_path):
    path = str(tmp_path / "checkpoints" / "global_step_2")
    os.makedirs(os.path.dirname(path))
    weights = {"actor_logstd": torch.full((1, 2), -0.5), "actor_mean.bias": torch.zeros(2)}
    trainer = {"actor": {"optimizer_steps": 8, "lr_scale": 0.25}, "fingerprint": _fp()}
    gen = torch.Generator().manual_seed(3).get_state()
    rank_state = {"global_step": 2, "env": {"counter": torch.tensor([7]), "reset_generator": gen}}
    os.makedirs(os.path.join(path, "stale"))  # an older checkpoint of the same step is replaced, not merged
    assert ckpt.write(path, 0, rank_state, weights, trainer) == path
    assert sorted(os.listdir(os.path.dirname(path))) == ["global_step_2"]  # no temporary directory left
    assert sorted(os.listdir(path)) == ["actor", "rank_0"]
    w = torch.load(os.path.join(path, "actor", "model_state_dict", "full_weights.pt"), weights_only=True)
    assert list(w) == list(weights) and all(torch.equal(w[k], weights[k]) for k in w)
    w2, t2, r2 = ckpt.read(path, 0)
    assert t2 == trainer and r2["global_step"] == 2 and torch.equal(r2["env"]["reset_generator"], gen)
    with pytest.raises(ValueError, match="ckpt_path"):
        ckpt.read(path, 1)
