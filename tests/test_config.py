import datetime as dt
import os

import pytest

from acco_b200.config import AttrDict, compose, default_config_dir, to_container

REF_TRAIN_KEYS = [  # every key of the reference's config/train/*.yaml
    "group_by_length", "batch_size", "n_grad_accumulation", "learning_rate", "weight_decay", "adam_beta1", "adam_beta2",
    "gradient_accumulation_steps", "nb_steps_tot", "dataloader_num_workers", "dataloader_pin_memory",
    "dataloader_persistent_workers", "label_smoothing_factor", "max_length", "scheduler_name", "warmup",
    "use_mixed_precision", "n_warmup_steps", "run_baseline_ddp", "method_name", "eval", "save", "eval_step",
    "run_expe_slow", "const_len_batch", "finetune",
]


def test_default_composition():
    cfg = compose()
    assert cfg.train.method_name == "acco"
    assert cfg.train.learning_rate == pytest.approx(6e-4) and isinstance(cfg.train.learning_rate, float)
    assert cfg.data.path == "Skylion007/openwebtext"
    assert cfg.model.arch == "llama" and cfg.model.hidden_size == 768
    assert cfg.run_name == "acco"
    for k in REF_TRAIN_KEYS:
        assert k in cfg.train, k


@pytest.mark.parametrize("name,method,bs,nacc,maxlen,ddp,nwarm", [
    ("acco", "acco", 8, 1, 1024, False, 0), ("dpu", "dpu", 8, 1, 1024, False, 1000), ("ddp", "ddp", 32, 1, 1024, True, 1000),
    ("acco-ft", "acco", 4, 2, 512, False, 0), ("dpu-ft", "dpu", 4, 4, 512, False, 50), ("ddp-ft", "ddp", 4, 4, 512, True, 0),
])
def test_train_groups_match_reference_values(name, method, bs, nacc, maxlen, ddp, nwarm):
    t = compose(overrides=[f"train={name}"]).train
    assert (t.method_name, t.batch_size, t.n_grad_accumulation, t.max_length, t.run_baseline_ddp, t.n_warmup_steps) == \
        (method, bs, nacc, maxlen, ddp, nwarm)
    assert t.const_len_batch == (not name.endswith("-ft"))
    assert t.finetune == name.endswith("-ft")


def test_overrides():
    cfg = compose(overrides=["train=ddp", "data=alpaca", "model=gptneo", "train.batch_size=4", "run_name=xp",
                             "+train.new_key=3.5", "train.learning_rate=1e-3", "train.slow_ranks=[1,3]"])
    assert cfg.train.method_name == "ddp" and cfg.train.batch_size == 4
    assert cfg.data.path == "tatsu-lab/alpaca"
    assert cfg.model.arch == "gptneo"
    assert cfg.run_name == "xp" and cfg.train.new_key == 3.5
    assert cfg.train.learning_rate == pytest.approx(1e-3)
    assert cfg.train.slow_ranks == [1, 3]
    assert cfg._groups_ == {"data": "alpaca", "train": "ddp", "model": "gptneo"}


def test_override_errors():
    with pytest.raises(KeyError):
        compose(overrides=["train.no_such_key=1"])
    with pytest.raises(FileNotFoundError):
        compose(overrides=["train=nope"])


def test_interpolation_and_container():
    cfg = compose(now=dt.datetime(2026, 1, 2, 3, 4, 5))
    assert cfg.hydra.run.dir == "./outputs/2026-01-02/03-04-05"
    plain = to_container(cfg.train)
    assert type(plain) is dict and plain["method_name"] == "acco"


def test_attrdict():
    a = AttrDict({"x": {"y": 1}, "l": [{"z": 2}]})
    assert a.x.y == 1 and a.l[0].z == 2
    a.x.y = 5
    assert a["x"]["y"] == 5
    b = a.copy()
    b.x.y = 6
    assert a.x.y == 5
    with pytest.raises(AttributeError):
        a.nope


def test_gptneo_json_present():
    assert os.path.isfile(os.path.join(default_config_dir(), "model", "gpt-neo-125M.json"))


def test_run_id_is_unique_outside_slurm_and_overridable(monkeypatch):
    """Two runs launched from one directory must not overwrite each other's checkpoints / TensorBoard dir
    (reference: `utils/logs_utils.py:19-40` create_id_run); Slurm job ids, ACCO_RUN_ID and a user-chosen --rdzv-id are kept."""
    from acco_b200.launch import DistEnv, _resolve_id, create_id_run, discover_env
    a, b = discover_env({}), discover_env({})
    _resolve_id(a), _resolve_id(b)
    assert a.id_run != "local" and len(a.id_run.split("_")) == 7 and (a.id_run != b.id_run or create_id_run() != create_id_run())
    assert discover_env({"ACCO_RUN_ID": "mine"}).id_run == "mine"
    tr = {"RANK": "0", "WORLD_SIZE": "1", "LOCAL_RANK": "0"}
    assert discover_env({**tr, "TORCHELASTIC_RUN_ID": "exp-7"}).id_run == "exp-7"
    e = discover_env({**tr, "TORCHELASTIC_RUN_ID": "none"})
    _resolve_id(e)
    assert e.id_run not in ("none", "torchrun") and len(e.id_run.split("_")) == 7
    assert discover_env({"SLURM_PROCID": "0", "SLURM_NTASKS": "1", "SLURM_JOBID": "4242"}).id_run == "4242"
    keep = DistEnv(id_run="job42")
    _resolve_id(keep)
    assert keep.id_run == "job42"


def test_launcher_topology_discovery():
    """Rank / node topology from the launcher's environment: Slurm (`trainer_base.py:137-151`: SLURM_{PROCID,LOCALID,NODEID,NTASKS,
    JOB_NODELIST,STEP_GPUS}, master = first host of the node list, port 12346 + lowest GPU id - numeric, not the reference's string
    min) and torchrun (RANK / LOCAL_RANK / LOCAL_WORLD_SIZE / GROUP_RANK)."""
    from acco_b200.launch import discover_env
    slurm = {"SLURM_PROCID": "11", "SLURM_LOCALID": "3", "SLURM_NODEID": "1", "SLURM_NTASKS": "16", "SLURM_JOBID": "777",
             "SLURM_JOB_NODELIST": "gpu[07-08]", "SLURM_STEP_GPUS": "10,9,2,3"}
    e = discover_env(slurm)
    assert (e.rank, e.local_rank, e.node_id, e.world_size, e.n_nodes) == (11, 3, 1, 16, 2)
    assert e.hostnames == ["gpu07", "gpu08"] and e.master_addr == "gpu07" and e.master_port == 12346 + 2 and e.launcher == "slurm"
    assert discover_env({**slurm, "MASTER_ADDR": "10.0.0.1", "MASTER_PORT": "5000"}).master_port == 5000
    tr = {"RANK": "13", "WORLD_SIZE": "16", "LOCAL_RANK": "5", "LOCAL_WORLD_SIZE": "8", "GROUP_RANK": "1", "MASTER_ADDR": "10.0.0.1",
          "MASTER_PORT": "29400", "TORCHELASTIC_RUN_ID": "exp"}
    t = discover_env(tr)
    assert (t.rank, t.local_rank, t.node_id, t.world_size, t.n_nodes, t.launcher) == (13, 5, 1, 16, 2, "torchrun")
    assert (t.master_addr, t.master_port, t.id_run) == ("10.0.0.1", 29400, "exp")
    # torchrun without the optional variables: one node assumed
    t1 = discover_env({"RANK": "3", "WORLD_SIZE": "4"})
    assert (t1.local_rank, t1.node_id, t1.n_nodes) == (3, 0, 1)
    single = discover_env({})
    assert (single.rank, single.world_size, single.launcher) == (0, 1, "single") and single.master_port > 0


def test_override_scalars_follow_hydra_not_yaml_1_1():
    """CLI overrides: PyYAML alone would turn `12:30` into 750 (base 60), `010` into 8 (octal) and `1_000` into 1000."""
    from acco_b200.config import _parse_value
    assert _parse_value("12:30") == "12:30" and _parse_value("1:24") == "1:24"
    assert _parse_value("010") == 10 and _parse_value("1_000") == "1_000"
    assert _parse_value("6e-4") == 6e-4 and _parse_value("3") == 3 and _parse_value("0.5") == 0.5 and _parse_value("-2") == -2
    assert _parse_value("true") is True and _parse_value("null") is None and _parse_value("[1,2]") == [1, 2]
    assert _parse_value("auto") == "auto" and _parse_value("1@24") == "1@24" and _parse_value("/data/ck_12:30.pt") == "/data/ck_12:30.pt"
