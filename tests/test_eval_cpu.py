"""CPU-side checks of the episode records and the evaluation calls (include/uavrl.h, uavrl_env_set_records, uavrl_eval_run): the
library exports them with the declared signatures, the record struct has the header's layout, and the Python layer turns
records into columns in slot / suite order."""
import ctypes as C

import numpy as np

import uavrl_b200  # noqa: F401
from uavrl_b200 import _lib, engine

NEW = ("uavrl_env_set_records", "uavrl_env_get_records", "uavrl_env_clear_records", "uavrl_eval_run", "uavrl_sac_eval_run",
       "uavrl_sac_act_mean")


def test_symbols_exported():
    L = _lib.lib()
    for s in NEW:
        assert hasattr(L, s) and s in _lib.SIGNATURES, s


def test_record_layout():
    """uavrl_episode_record: 8 int32 then 6 doubles, 80 bytes; uavrl_eval_stats: 3 int64"""
    R = _lib.EpisodeRecord
    assert C.sizeof(R) == 80 and C.sizeof(_lib.EvalStats) == 24
    assert R.total_score.offset == 32 and R.energy.offset == 72
    assert [f for f, _ in R._fields_][:8] == ["scenario", "env", "ordinal", "outcome", "steps", "subgoals", "collisions", "reserved"]


def test_argument_refusals_without_gpu():
    L = _lib.lib()
    assert L.uavrl_env_set_records(None, 4) == -1
    assert L.uavrl_eval_run(None, None, 0, 4, 0, None, None, None) == -1
    assert L.uavrl_sac_eval_run(None, None, 0, 4, 0, 0, None, None, None) == -1


def synthetic(n, N, G, done):
    buf = (_lib.EpisodeRecord * n)()
    for k in range(n):
        if k in done:
            buf[k].scenario, buf[k].env, buf[k].ordinal = 100 + k, k % N, k // N
            buf[k].outcome, buf[k].steps, buf[k].path_len = 1 + k % 2, 10 + k, 0.5 * k
    return buf


def test_record_columns_keep_written_slots():
    buf = synthetic(6, 4, 1, {0, 2, 5})
    out = engine.records_columns(buf, 6)
    assert list(out["slot"]) == [0, 2, 5] and list(out["env"]) == [0, 2, 1] and list(out["ordinal"]) == [0, 0, 1]
    assert list(out["steps"]) == [10, 12, 15] and out["path_len"].dtype == np.float64


def test_eval_result_suite_order_and_trainer():
    class Env:
        n = 8

    class Lrn:
        G = 4

    buf = synthetic(10, 8, 4, set(range(9)))
    st = _lib.EvalStats(30, 9, 1)
    res = engine._eval_result(Env(), Lrn(), 10, buf, st)
    r = res["records"]
    assert list(r["env"][:9]) == [k % 8 for k in range(9)]
    assert list(r["trainer"]) == [(k % 8) // 2 for k in range(9)] + [-1]
    assert r["outcome"][9] == 0 and (res["iterations"], res["n_records"], res["unfinished"]) == (30, 9, 1)


def test_plugin_summary_and_csv(tmp_path):
    import csv
    from uavrl_b200.plugins.PathPlan_City_B200 import eval_summary, write_eval_csv
    rec = {k: np.zeros(5) for k in engine.RECORD_FIELDS}
    rec["outcome"] = np.array([1, 2, 1, 0, 1], np.int32)
    rec["steps"] = np.array([10, 20, 30, 99, 40], np.int32)
    rec["path_len"] = np.array([12.0, 5.0, 30.0, 1.0, 8.0])
    rec["planner_len"] = np.array([10.0, 4.0, 20.0, 1.0, 0.0])
    rec["collisions"] = np.array([1, 0, 2, 7, 0], np.int32)
    rec["trainer"] = np.array([0, 0, 1, -1, 1])
    s = eval_summary(rec, num_trainers=2)
    assert (s["episodes"], s["success"], s["lose"], s["collisions"]) == (4, 3, 1, 3)
    assert s["success_rate"] == 0.75 and s["steps"] == 25.0 and s["path_len"] == 13.75
    assert s["path_ratio"] == (1.2 + 1.5) / 2                    # successful episodes with a planner path only
    assert s["success_rate_per_trainer"] == [0.5, 1.0]
    assert "success_rate_per_trainer" not in eval_summary(rec, 1)
    path = str(tmp_path / "logs" / "eval.csv")
    write_eval_csv(rec, path)
    rows = list(csv.reader(open(path)))
    assert rows[0][:3] == ["position", "scenario", "env"] and [r[0] for r in rows[1:]] == ["0", "1", "2", "4"]
