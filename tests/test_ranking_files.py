"""Ranking on file lists read by the actors (RayDMatrix(files, qid="qid"), distributed loading), on CPU: every file's
rows in stable qid order, one row block per file, rank-local group numbers as qid, the union of the ranks' groups equal
to the central matrix's, the refusals, and the driver-side check and prediction order through spawned actors.

The CPU stand-in engine (tests/cpu_engine.py) does not train with query groups, so training with the rank objectives
is left to tests/test_gpu_ranking_files.py; here the actors only carry a regression model through train / predict."""
import numpy as np
import pytest

from xgboost_ray_b200.matrix import RayDMatrix, RayDeviceQuantileDMatrix, RayShardingMode, group_offsets

N_FILES = 4
FEATURES = ["a", "b", "c", "d", "e"]


def make_frame(seed=0, n_groups=26):
    """One frame of query groups: qid = 1000 + 7 g (group g in file g mod 4, so the ids of the files interleave but
    are disjoint), group sizes 1..12 with one single-row group, 5 features with NaNs, labels 0..4."""
    import pandas as pd
    rng = np.random.RandomState(seed)
    sizes = rng.randint(2, 13, n_groups)
    sizes[5] = 1
    g = np.repeat(np.arange(n_groups), sizes)
    n = len(g)
    X = rng.normal(size=(n, len(FEATURES))).astype(np.float32)
    X[rng.rand(n, len(FEATURES)) < 0.1] = np.nan
    df = pd.DataFrame(X, columns=FEATURES)
    df["y"] = rng.randint(0, 5, n).astype(np.float32)
    df["qid"] = (1000 + 7 * g).astype(np.float32)
    df["file"] = g % N_FILES
    return df.iloc[rng.permutation(n)].reset_index(drop=True)        # rows unsorted inside every file


def write_files(tmp_path, df, fmt, name="part"):
    """The frame split into 4 files by its `file` column; the last file is written already sorted by qid."""
    files = []
    for i in range(N_FILES):
        part = df[df["file"] == i].drop(columns="file")
        if i == N_FILES - 1:
            part = part.sort_values("qid", kind="mergesort")
        f = str(tmp_path / ("%s%d.%s" % (name, i, fmt)))
        part.to_parquet(f, index=False) if fmt == "parquet" else part.to_csv(f, index=False)
        files.append(f)
    return files


def local_groups(shard):
    """The query groups of one shard: a list of (feature rows, labels) per group, from its rank-local qid."""
    q = np.asarray(shard["qid"])
    off = group_offsets(q)
    assert q.dtype == np.float32 and np.array_equal(np.unique(q), np.arange(len(off) - 1, dtype=np.float32))
    d = np.concatenate([np.asarray(b) for b in shard["data"]]) if isinstance(shard["data"], list) else np.asarray(shard["data"])
    return [(d[a:b], np.asarray(shard["label"])[a:b]) for a, b in zip(off[:-1], off[1:])]


def group_key(g):
    return g[0].tobytes() + g[1].tobytes()


@pytest.mark.parametrize("fmt", ["parquet", "csv"])
@pytest.mark.parametrize("actors", [1, 2, 3])
def test_shards_sort_each_file_and_keep_groups_whole(tmp_path, fmt, actors):
    files = write_files(tmp_path, make_frame(), fmt)
    m = RayDMatrix(files, label="y", qid="qid")
    assert m.distributed
    m.load_data(actors)
    # the central layout of each file on its own: what _load_groups makes of the same rows
    central_files = [RayDMatrix(f, label="y", qid="qid", distributed=False, num_actors=1).get_data(0) for f in files]
    assert np.any(np.diff(central_files[0]["qid"]) != 0)
    got_groups = []
    for r in range(actors):
        shard = m.get_data(r, actors)
        mine = list(range(r, N_FILES, actors))
        blocks = shard["data"] if isinstance(shard["data"], list) else [shard["data"]]
        assert len(blocks) == len(mine)                                   # one row block per file
        for b, i in zip(blocks, mine):
            assert np.array_equal(np.asarray(b), np.asarray(central_files[i]["data"]), equal_nan=True)
        assert all(np.asarray(b).shape[1] == len(FEATURES) for b in blocks)       # qid is not a feature
        want_label = np.concatenate([central_files[i]["label"] for i in mine])
        assert np.array_equal(shard["label"], want_label)
        # the rank-local group number: the files' central group numbers, offset file by file
        want_q, base = [], 0
        for i in mine:
            q = np.asarray(central_files[i]["qid"])
            want_q.append(q + base)
            base += len(group_offsets(q)) - 1
        assert np.array_equal(shard["qid"], np.concatenate(want_q))
        assert shard["qid"].dtype == np.float32
        got_groups += local_groups(shard)
    # the union of the ranks' groups is the central matrix's, with the same rows per group
    central = RayDMatrix(files, label="y", qid="qid", distributed=False, num_actors=1).get_data(0)
    want_groups = local_groups(central)
    assert len(got_groups) == len(want_groups) == 26
    assert sorted(map(group_key, got_groups)) == sorted(map(group_key, want_groups))
    assert min(len(g[1]) for g in got_groups) == 1                        # the single-row group
    # the prediction order: the files in list order, each one qid-sorted
    rows = np.concatenate(m._row_index)
    assert np.array_equal(np.sort(rows), np.arange(len(rows)))
    n = [len(c["label"]) for c in central_files]
    for r in range(actors):
        want = np.concatenate([np.arange(sum(n[:i]), sum(n[:i + 1])) for i in range(r, N_FILES, actors)])
        assert np.array_equal(m._row_index[r], want)


def test_batch_sharding_deals_consecutive_files(tmp_path):
    files = write_files(tmp_path, make_frame(1), "parquet")
    m = RayDMatrix(files, label="y", qid="qid", sharding=RayShardingMode.BATCH)
    m.load_data(2)
    one = RayDMatrix(files, label="y", qid="qid", num_actors=1).get_data(0)
    s0, s1 = m.get_data(0, 2), m.get_data(1, 2)
    assert np.array_equal(np.concatenate([s0["label"], s1["label"]]), one["label"])
    assert np.array_equal(np.concatenate(m._row_index), np.arange(len(one["label"])))


@pytest.mark.parametrize("fmt", ["parquet", "csv"])
def test_refusals(tmp_path, fmt):
    df = make_frame(2)
    files = write_files(tmp_path, df, fmt)
    # a qid shared by two files: the message names both files and the shared id
    shared = df.copy()
    shared.loc[shared.index[shared["qid"] == 1000 + 7 * 2][0], "file"] = 0     # one row of group 2 (file 2) into file 0
    bad = write_files(tmp_path, shared, fmt, name="shared")
    with pytest.raises(ValueError, match="query id 1014 appears in two files") as e:
        RayDMatrix(bad, label="y", qid="qid").load_data(2)
    assert repr(bad[0]) in str(e.value) and repr(bad[2]) in str(e.value)
    # an array qid cannot be split among the files
    with pytest.raises(ValueError, match="cannot be split among the files"):
        RayDMatrix(files, label="y", qid=df["qid"].values)
    with pytest.raises(ValueError, match="must be the name of a column"):
        RayDMatrix(files, label="y", qid=df["qid"].values, distributed=True)
    # still refused exactly as with central loading
    with pytest.raises(NotImplementedError, match="per-group weight"):
        RayDMatrix(files, label="y", qid="qid", weight="a")
    with pytest.raises(ValueError, match="use `qid` parameter instead"):
        RayDMatrix(files, label="y", group=[1, 2])
    with pytest.raises(ValueError, match="does not support ranking"):
        RayDeviceQuantileDMatrix(files, label="y", qid="qid")
    # a file list without qid is unchanged: no sorting, no qid, the prediction order is not set
    m = RayDMatrix(files, label="y")
    m.load_data(2)
    assert m.get_data(0, 2)["qid"] is None and m._row_index is None and not m._file_groups


@pytest.fixture
def cpu_actors(monkeypatch):
    """The CPU stand-in engine in the driver and, through a distributed callback, in every actor process."""
    import tests.cpu_engine as ce
    import xgboost_ray_b200.main as M
    import xgboost_ray_b200.xgb as seam
    monkeypatch.setenv("OMP_NUM_THREADS", "1")
    monkeypatch.setattr(seam, "xgboost", ce)
    orig = M._validate_ray_params

    def with_cpu_engine(rp):
        rp = orig(rp)
        rp.distributed_callbacks = [ce.UseCpuEngine()] + [c for c in (rp.distributed_callbacks or [])
                                                          if not isinstance(c, ce.UseCpuEngine)]
        return rp

    monkeypatch.setattr(M, "_validate_ray_params", with_cpu_engine)
    yield ce
    M.shutdown_actors()


@pytest.mark.timeout(600)
def test_actors_read_the_files_and_the_driver_checks_them(tmp_path, cpu_actors):
    """Through spawned actors: the driver refuses a qid shared by two files of the training or of an evaluation
    matrix before the first round, and predict returns the files in list order, each file's rows qid-sorted."""
    from xgboost_ray_b200 import RayParams, predict, train
    ce = cpu_actors
    df = make_frame(3)
    files = write_files(tmp_path, df, "parquet")
    shared = df.copy()
    shared.loc[shared.index[shared["qid"] == 1000 + 7 * 3][0], "file"] = 1     # group 3 (file 3) also in file 1
    bad = write_files(tmp_path, shared, "parquet", name="shared")
    params = {"objective": "reg:squarederror", "max_depth": 3, "nthread": 1}
    with pytest.raises(ValueError, match="query id 1021 appears in two files") as e:
        train(params, RayDMatrix(bad, label="y", qid="qid"), num_boost_round=2, ray_params=RayParams(num_actors=2))
    assert repr(bad[1]) in str(e.value) and repr(bad[3]) in str(e.value)
    with pytest.raises(ValueError, match="appears in two files"):
        train(params, RayDMatrix(files, label="y", qid="qid"), num_boost_round=2,
              evals=[(RayDMatrix(bad, label="y", qid="qid"), "v")], ray_params=RayParams(num_actors=2))
    extra = {}
    bst = train(params, RayDMatrix(files, label="y", qid="qid"), num_boost_round=3, additional_results=extra,
                ray_params=RayParams(num_actors=2))
    assert extra["total_n"] == len(df)
    sorted_files = [df[df["file"] == i].sort_values("qid", kind="mergesort") for i in range(N_FILES)]
    X = np.concatenate([f[FEATURES].to_numpy(np.float32) for f in sorted_files])
    want = bst.predict(ce.DMatrix(X))
    for actors in (1, 2, 3):
        got = predict(bst, RayDMatrix(files, qid="qid"), ray_params=RayParams(num_actors=actors))
        assert np.array_equal(got, want), actors
