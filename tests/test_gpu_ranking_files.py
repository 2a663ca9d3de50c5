"""GPU checks of ranking on file lists read by the actors (RayDMatrix(files, qid="qid")): for rank:pairwise, rank:ndcg
and rank:map on Parquet and CSV file lists, with 1 and 2 actors, the model is byte-identical to the one trained on the
central RayDMatrix of the same files, the ndcg / map / pre values of a file-list evaluation set equal the central ones,
predictions come back file by file with each file's rows in stable qid order, and a checkpoint restart gives the
uninterrupted model."""
import os

import numpy as np
import pytest

from tests.cpu_engine import TrainingCallback

pytestmark = pytest.mark.gpu

N_FILES = 4
FEATURES = ["f%d" % i for i in range(8)]
OBJECTIVES = ["rank:pairwise", "rank:ndcg", "rank:map"]
METRICS = ["ndcg@5", "map", "pre@3"]


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def make_frame(seed, n_groups):
    """Query groups of 1..80 rows (one single-row group) with qid = 11 + 3 g; group g goes to file g mod 4, so the
    files' ids interleave but are disjoint.  8 features with 5 % NaN, binary relevance labels that follow feature 0.
    Rows are shuffled, so no file is sorted by qid."""
    import pandas as pd
    rng = np.random.RandomState(seed)
    sizes = rng.randint(2, 81, n_groups)
    sizes[3] = 1
    g = np.repeat(np.arange(n_groups), sizes)
    n = len(g)
    X = rng.normal(size=(n, len(FEATURES))).astype(np.float32)
    y = (X[:, 0] + 0.7 * rng.normal(size=n) > 0.8).astype(np.float32)
    X[rng.rand(n, len(FEATURES)) < 0.05] = np.nan
    df = pd.DataFrame(X, columns=FEATURES)
    df["y"] = y
    df["qid"] = (11 + 3 * g).astype(np.float32)
    df["file"] = g % N_FILES
    return df.iloc[rng.permutation(n)].reset_index(drop=True)


def write_files(path, df, fmt, name):
    files = []
    for i in range(N_FILES):
        part = df[df["file"] == i].drop(columns="file")
        f = os.path.join(path, "%s%d.%s" % (name, i, fmt))
        part.to_parquet(f, index=False) if fmt == "parquet" else part.to_csv(f, index=False)
        files.append(f)
    return files


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("ranking_files"))
    train_df, eval_df = make_frame(0, 400), make_frame(1, 120)
    return {fmt: (write_files(path, train_df, fmt, "train"), write_files(path, eval_df, fmt, "eval"))
            for fmt in ("parquet", "csv")}


def file_list_order(file_list):
    """Positions, in the central (globally qid-sorted) prediction order, of the rows in the documented file-list
    order: the files in list order, each file's rows in stable qid order."""
    import pandas as pd
    read = (lambda f: pd.read_parquet(f)) if file_list[0].endswith(".parquet") else pd.read_csv
    qids = [read(f)["qid"].to_numpy(np.float32) for f in file_list]
    start = np.cumsum([0] + [len(q) for q in qids])
    central = np.argsort(np.concatenate(qids), kind="mergesort")      # central position -> row of the concatenation
    where = np.empty_like(central)
    where[central] = np.arange(len(central))
    rows = np.concatenate([start[i] + np.argsort(q, kind="mergesort") for i, q in enumerate(qids)])
    return where[rows]


def params_for(objective):
    return {"objective": objective, "max_depth": 6, "eta": 0.3, "lambdarank_num_pair_per_sample": 8,
            "eval_metric": METRICS}


def dump(bst):
    return bst.get_dump(dump_format="json", with_stats=True)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("actors", [1, 2])
@pytest.mark.parametrize("fmt", ["parquet", "csv"])
@pytest.mark.parametrize("objective", OBJECTIVES)
def test_file_list_equals_central(eng, files, objective, fmt, actors):
    if actors > eng.device_count():
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    train_files, eval_files = files[fmt]
    params = params_for(objective)
    res_c, res_f = {}, {}
    central = train(params, RayDMatrix(train_files, label="y", qid="qid", distributed=False), num_boost_round=6,
                    evals=[(RayDMatrix(eval_files, label="y", qid="qid", distributed=False), "v")], evals_result=res_c,
                    ray_params=RayParams(num_actors=1))
    dtrain = RayDMatrix(train_files, label="y", qid="qid")
    assert dtrain.distributed
    bst = train(params, dtrain, num_boost_round=6, evals=[(RayDMatrix(eval_files, label="y", qid="qid"), "v")],
                evals_result=res_f, ray_params=RayParams(num_actors=actors))
    assert not dtrain.refs                                               # the driver never read the rows
    assert len(dump(central)) == 6 and any('"split"' in t for t in dump(central))
    assert dump(bst) == dump(central)
    assert sorted(res_f["v"]) == sorted(METRICS) and all(len(v) == 6 for v in res_f["v"].values())
    assert res_f == res_c
    p_c = predict(central, RayDMatrix(train_files, qid="qid", ignore=["y"], distributed=False),
                  ray_params=RayParams(num_actors=1))
    p_f = predict(bst, RayDMatrix(train_files, qid="qid", ignore=["y"]), ray_params=RayParams(num_actors=actors))
    want = p_c[file_list_order(train_files)]
    assert p_f.dtype == want.dtype and p_f.tobytes() == want.tobytes()


class FailOnceCallback(TrainingCallback):
    """Raises in the actor after round `at` (once, guarded by a lock file): the driver restarts the attempt from its
    last checkpoint."""

    def __init__(self, lockfile, at):
        self.lockfile, self.at = lockfile, at

    def after_iteration(self, model, epoch, evals_log):
        if epoch == self.at and not os.path.exists(self.lockfile):
            with open(self.lockfile, "w") as f:
                f.write("failed")
            raise RuntimeError("training interrupted after round %d" % epoch)
        return False


@pytest.mark.timeout(600)
def test_checkpoint_restart_on_a_file_list(eng, files, tmp_path):
    """The attempt fails after round 4 (epoch 3) of 6; the driver restarts from the checkpoint of epoch 2 and the
    actor keeps the shard it read: the model equals the uninterrupted one."""
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    train_files, _ = files["parquet"]
    params = dict(params_for("rank:ndcg"), eval_metric="ndcg@5")
    ref = train(params, RayDMatrix(train_files, label="y", qid="qid"), num_boost_round=6,
                ray_params=RayParams(num_actors=1, checkpoint_frequency=2))
    lock = str(tmp_path / "lock")
    bst = train(params, RayDMatrix(train_files, label="y", qid="qid"), num_boost_round=6,
                ray_params=RayParams(num_actors=1, max_actor_restarts=1, checkpoint_frequency=2),
                callbacks=[FailOnceCallback(lock, at=3)])
    assert os.path.exists(lock)
    assert bst.num_boosted_rounds() == 6
    assert dump(bst) == dump(ref)
