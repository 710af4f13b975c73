"""Sampled Shapley attribution (lstm/shapley.py sampled_shapley, csrc/shapley.cu tb2_shapley_sample_*): the instance
plan and the phi / se reduction against NumPy / float64 restatements and the CLI refusals on the CPU; on the GPU the
permutations, every instance's value against the exact path's value of the same coalition, the reduction, agreement with
the exact values, null players, scenes beyond 12 players and the CLI."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_shapley import KINDS, _block, _model, _scene_batch, _scenes, _tc, _tree, instance_rows, select_players  # noqa: E402


# ---------------------------------------------------------------------------------------------------------------------
# restatements
# ---------------------------------------------------------------------------------------------------------------------
def sampled_instances(K, perms):
    """The coalition (set of ranks) of each instance of a scene with K players and permutations perms [P, >= K]."""
    if K == 0:
        return [set()]
    out = [set(), set(range(K))]
    for p in range(len(perms)):
        for k in range(1, K):
            out.append(set(int(r) for r in perms[p, :k]))
    return out


def reduce_ref(values, perms, K):
    """(phi [K], se [K]) of one metric from the scene's instance values [I] and permutations [P, >= K]: the module
    docstring's sums, float64, ascending pair order."""
    P = len(perms)
    Q = P // 2

    def v(p, k):
        return float(values[0 if k == 0 else 1 if k == K else 2 + p * (K - 1) + k - 1])

    phi, se = np.full(K, np.nan), np.full(K, np.nan)
    for j in range(K):
        a = []
        for q in range(Q):
            m = []
            for p in (2 * q, 2 * q + 1):
                k = list(perms[p, :K]).index(j)
                m.append(v(p, k + 1) - v(p, k))
            a.append((m[0] + m[1]) * 0.5)
        s = 0.0
        for x in a:
            s = s + x
        phi[j] = s / float(Q)
        d2 = 0.0
        for x in a:
            d = x - phi[j]
            d2 = d2 + d * d
        se[j] = math.sqrt(d2 / (float(Q) * float(Q - 1)))
    return phi, se


def _mask(ranks):
    return sum(1 << int(r) for r in ranks)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("players", [0, 1, 2, 5, None])
def test_sampled_plan_matches_the_restatement(players):
    from trajnetplusplusbaselines_b200.lstm.shapley import (_chunks_of, num_players, sampled_instance_counts,
                                                           sampled_instance_split)
    P = 6
    sizes = [1, 2, 3, 6, 7, 16, 31]                       # the last two have more than 12 neighbours
    obs, split = _scene_batch(3, sizes)
    K = num_players(sizes, 6143 if players is None else players)
    rs = np.random.RandomState(1)
    counts, rows = [], []
    for b, n in enumerate(sizes):
        k = int(K[b])
        assert k == (n - 1 if players is None else min(players, n - 1))
        prows = select_players(obs[-1, split[b]:split[b + 1]], k)
        perms = np.stack([rs.permutation(k) for _ in range(P)]) if k else np.zeros((P, 0), dtype=np.int64)
        inst = sampled_instances(k, perms)
        assert len(inst) == (1 if k == 0 else 2 + P * (k - 1))
        counts.append(len(inst))
        for coal in inst:
            r = instance_rows(n, prows, _mask(coal))
            assert r[0] == 0 and r == sorted(r)
            rows.append(len(r))
    assert np.array_equal(sampled_instance_counts(K, P), counts)
    assert np.array_equal(sampled_instance_split(sizes, K, P), np.concatenate([[0], np.cumsum(rows)]))
    for c in (max(counts), 100, 10 ** 6):
        parts = _chunks_of(counts, c)
        assert parts[0][0] == 0 and parts[-1][1] == len(sizes)
        assert all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
        assert all(sum(counts[b0:b1]) <= max(c, max(counts)) for b0, b1 in parts)


@pytest.mark.parametrize("K", [1, 2, 5, 13])
def test_reduction_restatement_and_efficiency(K):
    rs = np.random.RandomState(K)
    P = 8
    first = np.stack([rs.permutation(K) for _ in range(P // 2)])
    perms = np.empty((P, K), dtype=np.int64)
    perms[0::2], perms[1::2] = first, first[:, ::-1]
    values = rs.randn(2 + P * (K - 1))
    phi, se = reduce_ref(values, perms, K)
    assert abs(phi.sum() - (values[1] - values[0])) <= 1e-12 * K * max(1.0, abs(values).max())
    assert np.all(se >= 0)
    if K == 1:
        assert phi[0] == values[1] - values[0] and se[0] == 0.0
    # an additive game: every marginal is the player's weight, so phi is exact and se is 0
    w = rs.randn(K)
    add = np.array([sum(w[r] for r in c) for c in sampled_instances(K, perms)])
    phi, se = reduce_ref(add, perms, K)
    assert np.allclose(phi, w, atol=1e-12) and np.all(se <= 1e-12)


@pytest.mark.parametrize("argv, word", [
    (["--permutations", "5"], "--permutations"),
    (["--permutations", "2"], "--permutations"),
    (["--players", "all"], "--permutations"),
    (["--players", "13"], "--players must be in 0..12"),
    (["--seed", "3"], "--permutations"),
    (["--permutations", "8", "--players", "6144"], "--players"),
    (["--permutations", "8", "--seed", "-1"], "--seed"),
    (["--permutations", "8", "--players", "12", "--chunk", "50"], "--chunk"),
])
def test_cli_refusals_come_first(tmp_path, monkeypatch, argv, word):
    from trajnetplusplusbaselines_b200.lstm import LSTM, LSTMPredictor
    from trajnetplusplusbaselines_b200.lstm.shapley import main
    monkeypatch.chdir(tmp_path)
    _block(str(tmp_path))
    LSTMPredictor(LSTM()).save({}, "m.pkl")
    before = _tree(str(tmp_path))

    def no_read(*args, **kwargs):
        raise AssertionError("a dataset file was read")

    monkeypatch.setattr("trajnetplusplusbaselines_b200.data.load_test_scenes_xy", no_read)
    with pytest.raises(SystemExit) as e:
        main(["--path", "synth", "--output", "m.pkl"] + argv)
    assert word in str(e.value.code)
    assert _tree(str(tmp_path)) == before


def test_refusals_in_the_library():
    from trajnetplusplusbaselines_b200.lstm import LSTM
    from trajnetplusplusbaselines_b200.lstm.shapley import sampled_shapley
    from trajnetplusplusbaselines_b200.sgan import SGAN, LSTMGenerator
    from test_shapley import OwnPool
    obs = torch.zeros(9, 3, 2)
    for model in (LSTM(goal_flag=True), SGAN(generator=LSTMGenerator()), LSTM(pool=OwnPool())):
        with pytest.raises(NotImplementedError):
            sampled_shapley(model, obs, np.zeros((1, 12, 2)), [0, 3])
    model = LSTM()
    for kw, word in ((dict(permutations=6.5), "permutations"), (dict(permutations=3), "permutations"),
                     (dict(permutations=2), "permutations"), (dict(permutations=True), "permutations"),
                     (dict(players=6144), "players"), (dict(players=-1), "players"), (dict(players=1.5), "players"),
                     (dict(seed=-1), "seed"), (dict(seed=0.5), "seed"), (dict(n_predict=0), "n_predict"),
                     (dict(permutations=8, players=3, chunk=9), "10 instances")):
        with pytest.raises(ValueError, match=word):
            sampled_shapley(model, obs, np.zeros((1, 12, 2)), [0, 3], **kw)
    with pytest.raises(ValueError, match="truth"):
        sampled_shapley(model, obs, np.zeros((1, 11, 2)), [0, 3])


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _check_identities(res, values):
    """phi / se equal the restatement applied to the returned values and permutations, bit for bit; efficiency."""
    first = np.concatenate([[0], np.cumsum([1 if k == 0 else 2 + res.permutations.shape[1] * (k - 1)
                                            for k in res.num_players])])
    for b in range(len(res.num_players)):
        K = int(res.num_players[b])
        v = values[first[b]:first[b + 1]]
        assert v[1 if K else 0, 0] == res.v_full_ade[b] and v[0, 0] == res.v_empty_ade[b]
        assert v[1 if K else 0, 1] == res.v_full_fde[b] and v[0, 1] == res.v_empty_fde[b]
        for col, phi, se in ((0, res.phi_ade, res.se_ade), (1, res.phi_fde, res.se_fde)):
            ref_phi, ref_se = reduce_ref(v[:, col], res.permutations[b], K)
            assert phi[b, :K].tobytes() == ref_phi.tobytes() and se[b, :K].tobytes() == ref_se.tobytes(), (b, col)
            assert np.isnan(phi[b, K:]).all() and np.isnan(se[b, K:]).all()
            full, empty = v[1 if K else 0, col], v[0, col]
            assert abs(phi[b, :K].sum() - (full - empty)) <= 1e-12 * max(K, 1) * max(1.0, abs(full), abs(empty))
        assert np.all(res.player_rows[b, K:] == -1)


@pytest.mark.gpu
def test_permutations():
    from scipy import stats
    from trajnetplusplusbaselines_b200.lstm.shapley import sampled_shapley_scenes
    model = _model("vanilla")
    xys = _scenes(51, [1, 2, 4, 9, 14, 3])
    truths = [xy[9:21, 0] for xy in xys]
    a = sampled_shapley_scenes(model, xys, truths, permutations=8, seed=5)
    for b in range(len(xys)):
        K = int(a.num_players[b])
        assert K == xys[b].shape[1] - 1
        for p in range(8):
            assert sorted(a.permutations[b, p, :K]) == list(range(K)) and np.all(a.permutations[b, p, K:] == -1)
        assert np.array_equal(a.permutations[b, 1::2, :K], a.permutations[b, 0::2, :K][:, ::-1])
    same = sampled_shapley_scenes(model, xys, truths, permutations=8, seed=5, chunk=max(2 + 8 * 12, 1))
    assert same.permutations.tobytes() == a.permutations.tobytes()
    other = sampled_shapley_scenes(model, xys, truths, permutations=8, seed=6)
    assert other.permutations[4].tobytes() != a.permutations[4].tobytes()
    # a scene's permutations depend on (seed, its index, P, K) only: not on the scenes after it
    alone = sampled_shapley_scenes(model, xys[:5], truths[:5], permutations=8, seed=5)
    assert alone.permutations.tobytes() == a.permutations[:5, :, :alone.permutations.shape[2]].tobytes()
    # uniformity at K = 3: 3000 pairs per scene over two scenes; the 6 orders of each first permutation, chi-square
    # with 5 degrees of freedom at p >= 1e-6 (a correct sampler fails with probability 1e-6 per scene)
    xy3 = _scenes(52, [4, 4])
    r = sampled_shapley_scenes(model, xy3, [xy[9:21, 0] for xy in xy3], permutations=6000, seed=1, chunk=1 << 20)
    for b in range(2):
        codes = r.permutations[b, 0::2, :3] @ np.array([9, 3, 1])
        counts = np.array([np.sum(codes == c) for c in (5, 7, 11, 15, 19, 21)])      # the 6 permutations of 0, 1, 2
        assert counts.sum() == 3000
        assert stats.chisquare(counts).pvalue >= 1e-6, counts


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("kind", KINDS)
def test_instances_equal_the_exact_paths(monkeypatch, kind, tc):
    """Every sampled instance's value equals, bit for bit, the exact path's value of the same coalition mask; positions
    are the exact path's full-scene forecast."""
    from trajnetplusplusbaselines_b200.lstm.shapley import sampled_shapley_scenes, shapley_scenes
    _tc(monkeypatch, tc)
    model = _model(kind)
    xys = _scenes(61, [1, 2, 4, 7, 12])
    truths = [xy[9:21, 0] for xy in xys]
    for norm in (False, True):
        ex = shapley_scenes(model, xys, truths, players=5, normalize_scene=norm, return_values=True)
        sa = sampled_shapley_scenes(model, xys, truths, players=5, permutations=4, seed=2, normalize_scene=norm,
                                    return_values=True)
        assert np.array_equal(sa.num_players, ex.num_players)
        assert np.array_equal(sa.player_rows, ex.player_rows[:, :sa.player_rows.shape[1]])
        efirst = np.concatenate([[0], np.cumsum(1 << ex.num_players)])
        i = 0
        for b in range(len(xys)):
            K = int(sa.num_players[b])
            for coal in sampled_instances(K, sa.permutations[b]):
                assert sa.values[i].tobytes() == ex.values[efirst[b] + _mask(coal)].tobytes(), (kind, tc, norm, b)
                i += 1
        assert i == len(sa.values)
        assert sa.positions.tobytes() == ex.positions.tobytes()
        _check_identities(sa, sa.values)


@pytest.mark.gpu
def test_reduction_is_the_restatement_and_chunk_free():
    from trajnetplusplusbaselines_b200.lstm.shapley import sampled_shapley_scenes
    model = _model("social_default")
    xys = _scenes(71, [5, 1, 13, 2, 9, 20])
    truths = [xy[9:21, 0] for xy in xys]
    a = sampled_shapley_scenes(model, xys, truths, players=None, permutations=10, seed=3, return_values=True)
    _check_identities(a, a.values)
    b = sampled_shapley_scenes(model, xys, truths, players=None, permutations=10, seed=3, chunk=2 + 10 * 18,
                               return_values=True)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


@pytest.mark.gpu
def test_agrees_with_the_exact_values():
    """At K = 8 and P = 4096, |phi - phi_exact| <= 6 se + 1e-12 for every player."""
    from trajnetplusplusbaselines_b200.lstm.shapley import sampled_shapley_scenes, shapley_scenes
    model = _model("directional")
    xys = _scenes(81, [12, 9, 15])
    truths = [xy[9:21, 0] for xy in xys]
    ex = shapley_scenes(model, xys, truths, players=8)
    sa = sampled_shapley_scenes(model, xys, truths, players=8, permutations=4096, seed=0, chunk=1 << 16)
    assert np.all(sa.num_players == 8)
    for phi, ref, se in ((sa.phi_ade, ex.phi_ade, sa.se_ade), (sa.phi_fde, ex.phi_fde, sa.se_fde)):
        assert np.all(np.abs(phi - ref[:, :8]) <= 6 * se + 1e-12), (phi - ref[:, :8], se)


@pytest.mark.gpu
def test_null_players():
    from trajnetplusplusbaselines_b200.lstm.shapley import sampled_shapley_scenes
    xys = _scenes(91, [6, 15, 3])
    res = sampled_shapley_scenes(_model("vanilla"), xys, [xy[9:21, 0] for xy in xys], permutations=16)
    for b in range(len(xys)):
        K = int(res.num_players[b])
        for a in (res.phi_ade, res.phi_fde, res.se_ade, res.se_fde):
            assert np.all(a[b, :K] == 0.0)


@pytest.mark.gpu
def test_beyond_twelve_players():
    """players=None on scenes of 30+ tracks: K = N - 1, the identities, positions = _forward_nograd of the scenes."""
    from trajnetplusplusbaselines_b200.lstm.shapley import sampled_shapley
    model = _model("nn_lstm")
    obs, split = _scene_batch(7, [31, 40, 1, 35], n_frames=9)
    rs = np.random.RandomState(0)
    truth = obs[-1, split[:-1]][:, None, :].astype(np.float64) + np.cumsum(rs.randn(4, 12, 2) * 0.1, axis=1)
    res = sampled_shapley(model, torch.from_numpy(obs), truth, split, players=None, permutations=8, seed=4,
                          return_values=True)
    res = type(res)(*(f.cpu().numpy() for f in res))
    assert list(res.num_players) == [30, 39, 0, 34]
    for b, n in enumerate([31, 40, 1, 35]):
        assert list(res.player_rows[b, :n - 1]) == select_players(obs[-1, split[b]:split[b + 1]], n - 1)
    _check_identities(res, res.values)
    with torch.no_grad():
        _, pos = model._forward_nograd(torch.from_numpy(obs), torch.from_numpy(split), None, 12, pad_to_batch_max=False)
    assert res.positions.tobytes() == pos.cpu().numpy().tobytes()


@pytest.mark.gpu
def test_cli_end_to_end(tmp_path, monkeypatch, capsys):
    from trajnetplusplusbaselines_b200.data import load_test_scenes_xy
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    from trajnetplusplusbaselines_b200.lstm.shapley import format_line, format_se_line, main, summary
    monkeypatch.chdir(tmp_path)
    _block(str(tmp_path), sizes=(3, 1, 5, 2, 24, 4))
    LSTMPredictor(_model("directional").cpu()).save({}, "dlstm.pkl")
    main(["--path", "synth", "--output", "dlstm.pkl", "--players", "all", "--permutations", "8", "--seed", "2"])
    out = capsys.readouterr().out
    rec = np.load("dlstm_shapley_playersall_perm8_seed2.npz")
    scenes = load_test_scenes_xy(os.path.join("DATA_BLOCK", "synth", "test_private", "synth.ndjson"))
    n = len(scenes)
    W = max(xy.shape[1] - 1 for xy, _ in scenes)
    assert n == 6 and list(rec["dataset"]) == ["synth"] * n and W > 12
    assert list(rec["scene_id"]) == [meta.scene_id for _, meta in scenes]
    for k in ("phi_ade", "phi_fde", "se_ade", "se_fde", "player_ids"):
        assert rec[k].shape == (n, W)
    for k in ("v_full_ade", "v_full_fde", "v_empty_ade", "v_empty_fde", "num_players"):
        assert rec[k].shape == (n,)
    for i, (xy, meta) in enumerate(scenes):
        K = xy.shape[1] - 1
        assert rec["num_players"][i] == K
        prows = select_players(np.asarray(torch.Tensor(xy[:9]).numpy())[-1], K)
        peds = [meta.pedestrian] + list(meta.neigh_ids)
        assert list(rec["player_ids"][i, :K]) == [peds[r] for r in prows]
        assert np.all(rec["player_ids"][i, K:] == -1) and np.isnan(rec["se_ade"][i, K:]).all()
        assert np.all(rec["se_ade"][i, :K] >= 0)
    r = {k: rec[k] for k in rec.files}
    for label in ("synth", "pooled"):
        assert format_line(label, summary(r["phi_ade"], r["v_full_ade"], r["v_empty_ade"], r["num_players"]),
                           summary(r["phi_fde"], r["v_full_fde"], r["v_empty_fde"], r["num_players"])) in out
        assert format_se_line(label, r) in out
