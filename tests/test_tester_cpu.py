"""BatchedPolicyTester (mapdn_b200.marl_runner) against the reference's own PGTester (utilities/tester.py).

scripts/make_tester_golden.py ran the unmodified PGTester on the reference's env with a reference MADDPG model
(tests/golden/ref_tester.npz). Here the batched tester drives the oracle restatement of the env (tests/tester_cases.py:
OracleRecordEnv) with the recorded policy answers: records, record lengths and batch_run statistics agree to 1e-11.
The CUDA leg is tests/test_tester_gpu.py."""
import json
import pickle

import numpy as np
import pytest

import tester_cases as TC
from mapdn_b200.marl_runner import BatchedPolicyTester

TOL = 1e-11


def _golden():
    return np.load(TC.GOLDEN)


def _tester(g, name):
    case = json.loads(str(g["cases"]))[name]
    net, prof = TC.build(case)
    env = TC.OracleRecordEnv(net, prof, case["env_args"], case["batch"])
    return case, BatchedPolicyTester(env, TC.ReplayPolicy(g, name, case))


@pytest.mark.parametrize("name", ["rnn_day", "mlp_days", "diverge"])
def test_batched_run_reproduces_the_reference_tester(name):
    g = _golden()
    case, tester = _tester(g, name)
    records, lengths = tester.test_run(case["days"], hour=case["hour"], interval=case["interval"])
    want_len = g[f"{name}/lengths"]
    assert lengths.tolist() == want_len.tolist()
    want = np.split(g[f"{name}/records"], np.cumsum(want_len)[:-1])
    for i, w in enumerate(want):
        got = records[i].numpy()
        assert np.abs(got[:len(w)] - w).max() < TOL, i
        assert np.all(np.isnan(got[len(w):]))
    assert tester.net.checked == int(want_len.sum() - len(want_len))        # every policy call of the reference answered
    if name == "diverge":
        assert want_len[0] < case["max_steps"] + 1 and want_len[1] == case["max_steps"] + 1
    if name == "rnn_day":
        assert want_len[0] == 480                                           # manual_reset + 479 steps (episode_limit 480)


def test_records_for_day_have_the_reference_structure():
    g = _golden()
    case, tester = _tester(g, "mlp_days")
    tester.test_run(case["days"], hour=case["hour"], interval=case["interval"])
    rec = tester.records_for_day(1)
    assert list(rec) == list(TC.RECORD_KEYS)
    n = int(g["mlp_days/lengths"][1])
    widths = [w for _, w in tester.env.record_slices.values()]
    for (k, v), w in zip(rec.items(), widths):
        assert isinstance(v, list) and len(v) == n and all(isinstance(x, np.ndarray) and x.shape == (w,) for x in v)
    back = pickle.loads(pickle.dumps(rec, pickle.HIGHEST_PROTOCOL))
    assert np.array_equal(np.concatenate(back["bus_voltage"]), np.concatenate(rec["bus_voltage"]))


def test_batched_batch_run_reproduces_the_reference_statistics():
    g = _golden()
    case, tester = _tester(g, "batch")
    stat = tester.test_batch_run(case["episodes"])
    info = g["batch/info"]
    from oracle.voltage_control_ref import INFO_KEYS
    for k, key in enumerate(INFO_KEYS):
        m, s2 = stat["mean_test_" + key]
        assert abs(m - g["batch/stat"][k, 0]) < TOL and abs(s2 - g["batch/stat"][k, 1]) < TOL, key
        assert abs(m - np.mean(info[:, k])) < TOL and abs(s2 - 2 * np.std(info[:, k])) < TOL, key
    assert tester.net.checked == len(info)
