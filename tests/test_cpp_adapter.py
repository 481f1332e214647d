"""The C++ host-side mirror of the reference's ALMTrajOpt interface (include/ualm_traj_opt.hpp)."""
import struct
import subprocess

import numpy as np
import pytest

from harness import build_driver


@pytest.fixture(scope="module")
def driver(built, tmp_path_factory):
    d = tmp_path_factory.mktemp("cpp")
    return build_driver("adapter_driver", d)


def _write_case(path, m, pb, i):
    oxy, oyaw, _, _ = pb.offsets()
    with open(path, "wb") as f:
        f.write(struct.pack("<5i", *m.shape, int(pb.N[i]), int(pb.M[i])))
        f.write(m.cells.tobytes())
        f.write(pb.bnd[i].astype(np.float64).tobytes())
        f.write(struct.pack("<d", float(pb.total_time[i])))
        f.write(pb.inner_xy[oxy[i]:oxy[i + 1]].astype(np.float64).tobytes())
        f.write(pb.inner_yaw[oyaw[i]:oyaw[i + 1]].astype(np.float64).tobytes())


def test_result_containers_and_mpc_message_export(built, tmp_path):
    """make_traj / Piece::getValue / locatePieceIdx / toSE2TrajMsg of include/ualm_traj_opt.hpp against hand-computed values
    (se2traj.hpp:106-118, 343-367, 682-695; plan_manager.cpp:151-185) -- host only."""
    exe = build_driver("msg_driver", tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "OK", r.stdout


def test_adapter_compiles_and_fails_loudly_without_gpu(driver, bumps_map, tmp_path):
    import torch
    from uneven_planner_b200 import problems
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    pb = problems.generate(bumps_map, 1, seed=1)
    case = str(tmp_path / "case.bin")
    _write_case(case, bumps_map, pb, 0)
    r = subprocess.run([driver, case], capture_output=True, text=True)
    assert r.returncode == 10 and "EXCEPTION" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
def test_adapter_matches_batch_api(driver, bumps_map, tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from uneven_planner_b200 import _lib, api, problems
    pb = problems.generate(bumps_map, 2, seed=1)
    case = str(tmp_path / "case.bin")
    _write_case(case, bumps_map, pb, 1)
    r = subprocess.run([driver, case], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.strip().splitlines()
    head = lines[0].split()
    opt = api.BatchALMTrajOpt().init(_lib.default_params()).set_environment(bumps_map)
    res, cxy, cyaw = opt.optimize(pb)
    _, _, ocx, _ = pb.offsets()
    assert int(head[1]) == res[1].ret_code and int(head[3]) == res[1].n_evals and float(head[5]) == res[1].inner_cost
    N = int(pb.N[1])
    c = cxy[ocx[1]:ocx[2]]
    # getTraj() carries the piece durations of the last evaluation (T1(i), se2traj.hpp:682-695): bit-identical to the oracle's and
    # (tests/test_ref_pin.py) to the reference build's
    import pyoracle as po
    r_o = po.solve_one(po.params_from(_lib.default_params()), po.OracleMap(bumps_map), pb, 1)[0]
    dur = [float(x) for x in lines[2].split()[1:]]
    assert dur[0] == res[1].piece_T_xy and dur[1] == res[1].piece_T_yaw
    tt = 0.0
    for _ in range(int(pb.N[1])):
        tt += dur[0]
    assert tt == res[1].total_T == r_o.total_T
    lines = lines[:2] + lines[3:]
    coeffs = np.array([float(x) for x in lines[2:2 + 12 * N]]).reshape(N, 2, 6)
    for i in range(N):
        for d in range(2):
            assert np.array_equal(coeffs[i, d][::-1], c[6 * i + d * 6 * N: 6 * i + 6 + d * 6 * N])   # highest power first
    start = [float(x) for x in lines[1].split()[1:]]
    assert np.allclose(start, pb.bnd[1][:2], atol=1e-12)


@pytest.fixture(scope="module")
def chain_driver(built, tmp_path_factory):
    d = tmp_path_factory.mktemp("cppchain")
    return build_driver("chain_driver", d)


def _write_chain_case(path, m, starts, goals):
    with open(path, "wb") as f:
        f.write(struct.pack("<4i", *m.shape, len(starts)))
        f.write(m.cells.tobytes())
        f.write(np.ascontiguousarray(np.hstack([starts, goals]), dtype=np.float64).tobytes())


def _chain_pairs(B=12):
    rng = np.random.default_rng(9)
    starts = np.column_stack([rng.uniform(-4.3, 4.3, B), rng.uniform(-4.3, 4.3, B), rng.uniform(-np.pi, np.pi, B)])
    goals = np.column_stack([rng.uniform(-4.3, 4.3, B), rng.uniform(-4.3, 4.3, B), rng.uniform(-np.pi, np.pi, B)])
    return starts, goals


def test_chain_driver_plans_on_the_host_and_fails_loudly_without_gpu(chain_driver, bumps_map, tmp_path):
    """planAndOptimizeBatch: the front-end half runs on host threads; without a CUDA device the optimizer half throws"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    starts, goals = _chain_pairs()
    case = str(tmp_path / "chain.bin")
    _write_chain_case(case, bumps_map, starts, goals)
    r = subprocess.run([chain_driver, case, "64"], capture_output=True, text=True)
    assert r.returncode == 10 and "EXCEPTION" in r.stdout and "CUDA" in r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [64, 32])
def test_chain_through_the_cpp_class_matches_the_c_abi(chain_driver, bumps_map, tmp_path, prec):
    """(start, goal) pairs -> planAndOptimizeBatch -> exportToMpcBatch through include/ualm_traj_opt.hpp equals the same chain through the C ABI from Python"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from uneven_planner_b200 import _lib, api, front_end
    starts, goals = _chain_pairs()
    case = str(tmp_path / "chain.bin")
    _write_chain_case(case, bumps_map, starts, goals)
    r = subprocess.run([chain_driver, case, str(prec)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.strip().splitlines()
    head = [int(x) for x in lines[0].split()[1:]]
    view = front_end.MapView(bumps_map, 0.8, 0.003)
    pb, packed, _ = front_end.plan_batch(view, starts, goals, nthreads=2)
    assert head[0] == pb.B and head[1:] == list(packed) and pb.B >= 4
    opt = api.BatchALMTrajOpt(precision=prec).init(_lib.default_params()).set_environment(bumps_map)
    res, cxy, cyaw = opt.optimize(pb)
    ex = opt.mpc_export(pb.N, pb.M)
    opt.close()
    _, _, ocx, _ = pb.offsets()
    sN = np.concatenate([[0], np.cumsum(pb.N)])
    for i in range(pb.B):
        v = lines[1 + i].split()
        assert (int(v[0]), int(v[1]), int(v[2]), int(v[3])) == (int(pb.N[i]), int(pb.M[i]), res[i].ret_code, res[i].n_evals)
        got = [float(x) for x in v[4:]]
        want = [res[i].inner_cost, cxy[ocx[i] + 1], ex["pos_pts"][2 * (sN[i] + i)], ex["c_mpc_xy"][ocx[i] + 3], ex["dev"][i, 0]]
        assert got == want, (i, got, want)
