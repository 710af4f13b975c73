"""Shapley attribution of forecast errors to neighbours (lstm/shapley.py, csrc/shapley.cu): the player selection, the
instance plan and the Shapley sum against NumPy / float64 restatements on the CPU; on the GPU the expansion kernel, the
instance forecasts and values against per-scene predictions and the scorer, the value kernel's sums, null players,
chunking and the CLI."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

MAX_PLAYERS = 12


# ---------------------------------------------------------------------------------------------------------------------
# restatements
# ---------------------------------------------------------------------------------------------------------------------
def select_players(last, players):
    """The player rows by rank for one scene: last [N, 2] float32 positions at the last observed frame, primary first.
    Squared distance in float64, +inf where not finite, ties to the lower row."""
    n = last.shape[0]
    K = min(players, max(n - 1, 0))
    x0, y0 = float(last[0, 0]), float(last[0, 1])
    dist = {}
    for j in range(1, n):
        dx, dy = float(last[j, 0]) - x0, float(last[j, 1]) - y0
        d = dx * dx + dy * dy
        dist[j] = d if math.isfinite(d) else math.inf
    return sorted(range(1, n), key=lambda j: (dist[j], j))[:K]


def instance_rows(n, player_rows, mask):
    """Rows of the scene kept by coalition `mask` (bit r = the player of rank r), in their original order."""
    deleted = {p for r, p in enumerate(player_rows) if not (mask >> r) & 1}
    return [j for j in range(n) if j not in deleted]


def shapley_ref(v, K):
    """phi [K] from the value table v [2^K] (mask order): ascending S over the subsets without j, float64, weights from
    exact factorials, term w * (v(S + j) - v(S)) added in that order."""
    phi = []
    for j in range(K):
        acc = 0.0
        for S in range(1 << K):
            if (S >> j) & 1:
                continue
            w = float(math.factorial(bin(S).count('1')) * math.factorial(K - bin(S).count('1') - 1)) / float(math.factorial(K))
            acc = acc + w * (float(v[S | (1 << j)]) - float(v[S]))
        phi.append(acc)
    return np.array(phi, dtype=np.float64)


def _scene_batch(seed, sizes, n_frames=9, nan_last=True, ties=True):
    """float32 observed [n_frames, M, 2] and split for scenes of `sizes`: a neighbour NaN at the last frame and two
    neighbours at the same position there."""
    rs = np.random.RandomState(seed)
    split = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    obs = (rs.randn(1, split[-1], 2) * 2.0 + np.cumsum(rs.randn(n_frames, split[-1], 2) * 0.2, axis=0)).astype(np.float32)
    for b, n in enumerate(sizes):
        r0 = split[b]
        if nan_last and n > 2:
            obs[-1, r0 + 1] = np.nan
        if ties and n > 4:
            obs[-1, r0 + 4] = obs[-1, r0 + 2]                            # same position: an exact distance tie
    return obs, split


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("players", [0, 1, 3, 8, 12])
def test_plan_matches_the_restatement(players):
    from trajnetplusplusbaselines_b200.lstm.shapley import chunks, instance_split, num_players
    sizes = [1, 2, 3, 5, 7, 13, 20]
    obs, split = _scene_batch(3, sizes)
    K = num_players(sizes, players)
    counts, rows_total = [], []
    for b, n in enumerate(sizes):
        prows = select_players(obs[-1, split[b]:split[b + 1]], players)
        assert len(prows) == K[b] == min(players, n - 1)
        for mask in range(1 << len(prows)):
            rows = instance_rows(n, prows, mask)
            assert rows[0] == 0 and rows == sorted(rows)
            counts.append(len(rows))
        rows_total.append(prows)
    assert np.array_equal(instance_split(sizes, K), np.concatenate([[0], np.cumsum(counts)]))
    for c in (1 << int(K.max()), 50, 4096):
        parts = chunks(K, c)
        assert parts[0][0] == 0 and parts[-1][1] == len(sizes)
        assert all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
        assert all(sum(1 << int(k) for k in K[b0:b1]) <= max(c, 1 << int(K.max())) for b0, b1 in parts)
    if players >= 4:
        # scene 4 (7 tracks): row 1 is NaN at the last frame and comes last; row 4 ties with row 2 and follows it
        prows = rows_total[4]
        assert prows.index(2) + 1 == prows.index(4)
        if players >= 6:
            assert prows[-1] == 1


def test_selection_edge_cases():
    nan = np.float32(np.nan)
    last = np.array([[0, 0], [1, 0], [0, 1], [nan, 0], [-1, 0], [0.5, 0.5]], dtype=np.float32)
    assert select_players(last, 12) == [5, 1, 2, 4, 3]                # ties to the lower row, NaN last
    assert select_players(last, 2) == [5, 1]
    assert select_players(last, 0) == []
    assert select_players(last[:1], 8) == []                          # N = 1
    assert instance_rows(6, [5, 1, 2], 0b010) == [0, 1, 3, 4]
    assert instance_rows(6, [5, 1, 2], 0b111) == list(range(6))


@pytest.mark.parametrize("K", [1, 2, 5, 9])
def test_shapley_sum_properties(K):
    rs = np.random.RandomState(K)
    base = rs.randn(1 << K)
    # efficiency on a random game
    phi = shapley_ref(base, K)
    assert abs(phi.sum() - (base[-1] - base[0])) < 1e-9
    # an additive game with two symmetric players (0 and 1) and a null player (the last)
    weights = rs.randn(K)
    if K >= 3:
        weights[1] = weights[0]
    weights[-1] = 0.0
    v = np.array([sum(weights[r] for r in range(K) if (m >> r) & 1) for m in range(1 << K)])
    # a symmetric interaction term between 0 and 1 keeps them symmetric
    if K >= 3:
        v = v + np.array([0.7 if (m & 3) == 3 else 0.0 for m in range(1 << K)])
    phi = shapley_ref(v, K)
    assert phi[-1] == 0.0
    assert abs(phi.sum() - (v[-1] - v[0])) < 1e-9
    if K >= 3:
        assert phi[0] == phi[1]
        assert abs(phi[0] - (weights[0] + 0.35)) < 1e-12


class OwnPool(torch.nn.Module):
    """A user-defined interaction module (no fill_config)."""

    def __init__(self, hidden_dim=128, out_dim=32):
        super().__init__()
        self.out_dim = out_dim
        self.linear = torch.nn.Linear(hidden_dim, out_dim)

    def reset(self, num_tracks, max_num_neigh, device):
        pass

    def forward(self, hidden, obs1, obs2):
        return self.linear(hidden).reshape(-1, self.out_dim)


def _block(root, name="synth", sizes=(3, 1, 5, 2, 7, 4)):
    from test_multimodal_batch import _write_scenes
    for part in ("test", "test_private"):
        os.makedirs(os.path.join(root, "DATA_BLOCK", name, part))
        _write_scenes(os.path.join(root, "DATA_BLOCK", name, part, name + ".ndjson"), list(sizes), 4)


def _tree(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


@pytest.mark.parametrize("which", ["goal", "sgan", "own", "players13"])
def test_cli_refusals_come_first(tmp_path, monkeypatch, which):
    from trajnetplusplusbaselines_b200.lstm import LSTM, LSTMPredictor
    from trajnetplusplusbaselines_b200.lstm.shapley import main
    from trajnetplusplusbaselines_b200.sgan import SGAN, SGANPredictor, LSTMGenerator
    monkeypatch.chdir(tmp_path)
    _block(str(tmp_path))
    argv = ["--path", "synth", "--output", "m.pkl"]
    if which == "goal":
        LSTMPredictor(LSTM(goal_flag=True)).save({}, "m.pkl")
        word = "goal"
    elif which == "sgan":
        SGANPredictor(SGAN(generator=LSTMGenerator())).save({}, "m.pkl")
        word = "SGAN"
    elif which == "own":
        LSTMPredictor(LSTM(pool=OwnPool())).save({}, "m.pkl")
        word = "OwnPool"
    else:
        argv += ["--players", "13"]
        word = "--players"
    before = _tree(str(tmp_path))
    with pytest.raises(SystemExit) as e:
        main(argv)
    assert word in str(e.value.code)
    assert _tree(str(tmp_path)) == before


def test_refusals_in_the_library():
    from trajnetplusplusbaselines_b200.lstm import LSTM
    from trajnetplusplusbaselines_b200.lstm.shapley import shapley
    from trajnetplusplusbaselines_b200.sgan import SGAN, LSTMGenerator
    obs = torch.zeros(9, 3, 2)
    for model in (LSTM(goal_flag=True), SGAN(generator=LSTMGenerator()), LSTM(pool=OwnPool()), LSTMGenerator()):
        with pytest.raises(NotImplementedError):
            shapley(model, obs, np.zeros((1, 12, 2)), [0, 3])
    model = LSTM()
    for kw in (dict(players=13), dict(players=-1), dict(players=2.5)):
        with pytest.raises(ValueError, match="players"):
            shapley(model, obs, np.zeros((1, 12, 2)), [0, 3], **kw)
    with pytest.raises(ValueError, match="n_predict"):
        shapley(model, obs, np.zeros((1, 12, 2)), [0, 3], n_predict=0)
    with pytest.raises(ValueError, match="truth"):
        shapley(model, obs, np.zeros((1, 11, 2)), [0, 3])
    bad = np.zeros((2, 12, 2))
    bad[1, 4, 0] = np.nan
    with pytest.raises(ValueError, match="scene 1"):
        shapley(model, torch.zeros(9, 4, 2), bad, [0, 3, 4])


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


@pytest.mark.gpu
@pytest.mark.parametrize("players", [0, 3, 8, 12])
def test_expansion_is_base_rows(players):
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm.shapley import instance_split, num_players
    lib = _lib.load()
    sizes = [1, 2, 3, 5, 7, 13, 20, 4]
    obs, split = _scene_batch(5, sizes)
    K = num_players(sizes, players)
    first = np.concatenate([[0], np.cumsum(1 << K)])
    isplit = instance_split(sizes, K)
    I, M_out = int(first[-1]), int(isplit[-1])
    dev = torch.device("cuda")
    i32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int32)).to(dev)
    base = torch.from_numpy(obs).to(dev)
    out = torch.full((obs.shape[0], M_out, 2), 7.0, device=dev)
    rows = torch.empty((len(sizes), MAX_PLAYERS), dtype=torch.int32, device=dev)
    coal = torch.empty(I, dtype=torch.int32, device=dev)
    scene_off, first_d, isplit_d = i32(split), i32(first), i32(isplit)
    before = lib.tb2_launch_count()
    _lib.check(lib.tb2_shapley_expand(_p(base), obs.shape[0], obs.shape[1], _p(scene_off), _p(first_d), _p(isplit_d),
                                      len(sizes), I, max(sizes), M_out, _p(out), _p(rows), _p(coal),
                                      ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert lib.tb2_launch_count() - before == 1
    out, rows, coal = out.cpu().numpy(), rows.cpu().numpy(), coal.cpu().numpy()
    for b, n in enumerate(sizes):
        scene = obs[:, split[b]:split[b + 1]]
        prows = select_players(scene[-1], players)
        assert list(rows[b, :len(prows)]) == prows and np.all(rows[b, len(prows):] == -1)
        for mask in range(1 << len(prows)):
            i = first[b] + mask
            assert coal[i] == mask
            want = scene[:, instance_rows(n, prows, mask)]
            got = out[:, isplit[i]:isplit[i + 1]]
            assert got.tobytes() == want.tobytes(), (b, mask)
    assert not (out == 7.0).all(axis=2).any()                            # every output row written


def _model(kind, seed=1):
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200.lstm import (AttentionMLPPooling, GridBasedPooling, HiddenStateMLPPooling, LSTM,
                                                    NearestNeighborLSTM, NearestNeighborMLP, TrajectronPooling)
    if kind in O.MODEL_SPECS:
        spec = O.MODEL_SPECS[kind]
        pool = GridBasedPooling(**spec) if spec is not None else None
    else:
        pool = {"hiddenstatemlp": lambda: HiddenStateMLPPooling(**O.NONGRID_SPECS[kind]),
                "nn": lambda: NearestNeighborMLP(**O.NN_SPECS[kind]),
                "attentionmlp": lambda: AttentionMLPPooling(**O.ATTN_SPECS[kind]),
                "nn_lstm": lambda: NearestNeighborLSTM(**O.NN_LSTM_SPECS[kind]),
                "traj_pool": lambda: TrajectronPooling(**O.TRAJ_SPECS[kind])}[kind]()
    model = LSTM(pool=pool)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=seed).items()})
    return model.cuda().eval()


def _scenes(seed, sizes):
    from oracle import lstm_oracle as O
    xys = []
    for i, n in enumerate(sizes):
        xy, _ = O.synthetic_scenes(1, n, n_frames=21, seed=seed * 100 + i, ragged=False, nan_tracks=False)
        xys.append(xy[:, :n].astype(np.float64))
    return xys


def _score(pred_primary, truth):
    """score_arrays' mode-0 ADE / FDE of primaries [S, T, 2] against truth [S, T, 2]."""
    from trajnetplusplusbaselines_b200 import scoring
    S, T = truth.shape[:2]
    z = np.zeros(S + 1, dtype=np.int32)
    a = dict(gt_primary=truth, pred_primary=np.asarray(pred_primary, dtype=np.float64)[:, None], num_modes=np.ones(S),
             gt_neigh_off=z, pred_neigh_off=z, gt_neigh=np.zeros((0, T, 2)), gt_neigh_mask=np.zeros((0, T)),
             pred_neigh=np.zeros((0, T, 2)), pred_neigh_mask=np.zeros((0, T)))
    r = scoring.score_arrays(a, False)
    return r["ade"][:, 0], r["fde"][:, 0]


def _tc(monkeypatch, tc):
    if tc:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    else:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")


KINDS = ["vanilla", "occupancy", "directional", "social_default", "social", "hiddenstatemlp", "nn", "attentionmlp",
         "nn_lstm", "traj_pool"]


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("kind", KINDS)
def test_instances_match_per_scene_predictions(monkeypatch, kind, tc):
    """For a sample of instances across scene sizes, the value of each is score_arrays' mode-0 ADE / FDE of
    predict_batch_xy's prediction of the reduced scene alone, bit for bit, and v(full) / v(empty) are those of the full
    scene and of the scene without its players; the full scenes' positions are _forward_nograd's."""
    from types import SimpleNamespace
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    from trajnetplusplusbaselines_b200.lstm.shapley import shapley_scenes
    _tc(monkeypatch, tc)
    model = _model(kind)
    sizes = [1, 2, 4, 7, 12, 20]
    xys = _scenes(11, sizes)
    truths = [xy[9:21, 0] for xy in xys]
    players = 4
    rs = np.random.RandomState(3)
    for norm in (False, True):
        res = shapley_scenes(model, xys, truths, players=players, normalize_scene=norm, return_values=True)
        first = np.concatenate([[0], np.cumsum(1 << res.num_players)])
        reduced, want_rows, want_truth = [], [], []
        for b, xy in enumerate(xys):
            K = int(res.num_players[b])
            prows = list(res.player_rows[b, :K])
            obs32 = np.asarray(torch.Tensor(xy[:9]).numpy()) if not norm else None
            if obs32 is not None:
                assert prows == select_players(obs32[-1], players)
            masks = sorted(set([0, (1 << K) - 1] + list(rs.randint(0, 1 << K, 3))))
            for m in masks:
                reduced.append(xy[:, instance_rows(xy.shape[1], prows, m)])
                want_rows.append(first[b] + m)
                want_truth.append(truths[b])
        pred = LSTMPredictor(model).predict_batch_xy(reduced, n_predict=12, args=SimpleNamespace(normalize_scene=norm))
        ade, fde = _score(np.stack([p[0][0] for p in pred]), np.stack(want_truth))
        got = res.values[want_rows]
        assert got[:, 0].tobytes() == ade.tobytes() and got[:, 1].tobytes() == fde.tobytes(), (kind, tc, norm)
        full = LSTMPredictor(model).predict_batch_xy(xys, n_predict=12, args=SimpleNamespace(normalize_scene=norm))
        fa, ff = _score(np.stack([p[0][0] for p in full]), np.stack(truths))
        assert res.v_full_ade.tobytes() == fa.tobytes() and res.v_full_fde.tobytes() == ff.tobytes()
        empty = [xy[:, instance_rows(xy.shape[1], list(res.player_rows[b, :res.num_players[b]]), 0)]
                 for b, xy in enumerate(xys)]
        pe = LSTMPredictor(model).predict_batch_xy(empty, n_predict=12, args=SimpleNamespace(normalize_scene=norm))
        ea, ef = _score(np.stack([p[0][0] for p in pe]), np.stack(truths))
        assert res.v_empty_ade.tobytes() == ea.tobytes() and res.v_empty_fde.tobytes() == ef.tobytes()
        if not norm:
            split = np.concatenate([[0], np.cumsum(sizes)])
            with torch.no_grad():
                _, pos = model._forward_nograd(torch.Tensor(np.concatenate([xy[:9] for xy in xys], axis=1)),
                                               torch.from_numpy(split), None, 12, pad_to_batch_max=False)
            assert res.positions.tobytes() == pos.cpu().numpy().tobytes()


@pytest.mark.gpu
def test_phi_is_the_restated_sum_of_the_kernels_values():
    from trajnetplusplusbaselines_b200.lstm.shapley import shapley_scenes
    model = _model("directional")
    xys = _scenes(21, [13, 5, 1, 9])
    truths = [xy[9:21, 0] for xy in xys]
    for players in range(0, 13):
        res = shapley_scenes(model, xys, truths, players=players, return_values=True)
        first = np.concatenate([[0], np.cumsum(1 << res.num_players)])
        for b in range(len(xys)):
            K = int(res.num_players[b])
            v = res.values[first[b]:first[b + 1]]
            assert v[-1, 0] == res.v_full_ade[b] and v[0, 0] == res.v_empty_ade[b]
            assert v[-1, 1] == res.v_full_fde[b] and v[0, 1] == res.v_empty_fde[b]
            for col, phi in ((0, res.phi_ade), (1, res.phi_fde)):
                ref = shapley_ref(v[:, col], K)
                assert phi[b, :K].tobytes() == ref.tobytes(), (players, b, col)
                assert np.isnan(phi[b, K:]).all()
                assert abs(phi[b, :K].sum() - (v[-1, col] - v[0, col])) <= 1e-9
            assert np.all(res.player_rows[b, K:] == -1)


@pytest.mark.gpu
def test_null_players():
    from trajnetplusplusbaselines_b200.lstm.shapley import shapley_scenes
    xys = _scenes(31, [6, 9, 3])
    truths = [xy[9:21, 0] for xy in xys]
    res = shapley_scenes(_model("vanilla"), xys, truths, players=5)
    for b in range(len(xys)):
        K = int(res.num_players[b])
        assert np.all(res.phi_ade[b, :K] == 0.0) and np.all(res.phi_fde[b, :K] == 0.0)
    # occupancy (cells of 0.6 m, 12 x 12): one neighbour walks parallel to the primary 100 m to its side, never in the
    # grid; another walks 1 m beside it
    t = np.arange(21, dtype=np.float64)
    prim = np.stack([0.4 * t, 0.05 * t], axis=1)
    xy = np.stack([prim, prim + [0.0, 1.0], prim + [0.0, 100.0]], axis=1)
    res = shapley_scenes(_model("occupancy"), [xy], [xy[9:21, 0]], players=2)
    rows = list(res.player_rows[0, :2])
    far, near = rows.index(2), rows.index(1)
    assert res.phi_ade[0, far] == 0.0 and res.phi_fde[0, far] == 0.0
    assert res.phi_ade[0, near] != 0.0


@pytest.mark.gpu
def test_results_do_not_depend_on_chunk():
    from trajnetplusplusbaselines_b200.lstm.shapley import shapley_scenes
    model = _model("social_default")
    xys = _scenes(41, [5, 8, 1, 3, 12, 6, 2])
    truths = [xy[9:21, 0] for xy in xys]
    a = shapley_scenes(model, xys, truths, players=3, chunk=65536, return_values=True)
    b = shapley_scenes(model, xys, truths, players=3, chunk=9, return_values=True)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


@pytest.mark.gpu
def test_cli_end_to_end(tmp_path, monkeypatch, capsys):
    from trajnetplusplusbaselines_b200.data import load_test_scenes_xy
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    from trajnetplusplusbaselines_b200.lstm.shapley import format_line, main, summary
    monkeypatch.chdir(tmp_path)
    _block(str(tmp_path))
    LSTMPredictor(_model("directional").cpu()).save({}, "dlstm.pkl")
    main(["--path", "synth", "--output", "dlstm.pkl", "--players", "3"])
    out = capsys.readouterr().out
    rec = np.load("dlstm_shapley_players3.npz")
    scenes = load_test_scenes_xy(os.path.join("DATA_BLOCK", "synth", "test_private", "synth.ndjson"))
    n = len(scenes)
    assert n == 6 and list(rec["dataset"]) == ["synth"] * n
    assert list(rec["scene_id"]) == [meta.scene_id for _, meta in scenes]
    for k in ("phi_ade", "phi_fde", "player_ids"):
        assert rec[k].shape == (n, MAX_PLAYERS)
    for k in ("v_full_ade", "v_full_fde", "v_empty_ade", "v_empty_fde", "num_players"):
        assert rec[k].shape == (n,)
    for i, (xy, meta) in enumerate(scenes):
        K = min(3, xy.shape[1] - 1)
        assert rec["num_players"][i] == K
        prows = select_players(np.asarray(torch.Tensor(xy[:9]).numpy())[-1], 3)
        peds = [meta.pedestrian] + list(meta.neigh_ids)
        assert list(rec["player_ids"][i, :K]) == [peds[r] for r in prows]
        assert np.all(rec["player_ids"][i, K:] == -1)
    assert rec["num_players"][1] == 0                                    # the scene with only its primary
    for label in ("synth", "pooled"):
        line = format_line(label, summary(rec["phi_ade"], rec["v_full_ade"], rec["v_empty_ade"], rec["num_players"]),
                           summary(rec["phi_fde"], rec["v_full_fde"], rec["v_empty_fde"], rec["num_players"]))
        assert line in out
    absphi = np.nan_to_num(np.abs(rec["phi_ade"]))
    assert ("%12.6f" % np.mean(absphi.sum(axis=1))) in out
    assert ("%12.6f" % np.mean(rec["v_empty_ade"] - rec["v_full_ade"])) in out
