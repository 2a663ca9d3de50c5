"""UBJSON model files on the GPU (DESIGN.md 2 item 25): a model saved as .ubj and loaded again reaches the existing
prediction, TreeSHAP, leaf-index and training paths with exactly the trees of the source model, so every output equals
the source's bit for bit, and continuing from the UBJSON file equals continuing from the JSON file."""
import json

import numpy as np
import pytest
import scipy.sparse as sp

from tests.test_gpu_model_slicing import BASE, CASES, ROUNDS, _assert_same, _data, _outputs
from tests.test_model_json import XGB_STYLE
from tests.test_model_ubjson import TYPED, Enc, dec

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def E():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


KINDS = list(CASES) + ["rank_ndcg", "csr"]


def _train_data(E, kind):
    """(params, train matrix, prediction matrix) of a model kind."""
    if kind == "rank_ndcg":
        rng = np.random.RandomState(4)
        sizes = rng.randint(2, 30, 150)
        qid = np.repeat(np.arange(len(sizes)), sizes)
        X = rng.uniform(0, 10, size=(len(qid), 8)).astype(np.float32)
        y = np.clip(np.round(X[:, 0] / 3 + rng.normal(size=len(qid))), 0, 3).astype(np.float32)
        params = dict(BASE, objective="rank:ndcg")
        return params, E.DMatrix(X, label=y, qid=qid), E.DMatrix(rng.uniform(0, 10, size=(600, 8)).astype(np.float32))
    if kind == "csr":
        rng = np.random.RandomState(5)
        X = sp.random(4000, 30, density=0.2, format="csr", random_state=rng, dtype=np.float32) * 10
        y = (np.asarray(X[:, 0].todense()).ravel() + np.asarray(X[:, 1].todense()).ravel() > 1).astype(np.float32)
        Xp = sp.random(700, 30, density=0.2, format="csr", random_state=rng, dtype=np.float32) * 10
        return dict(BASE, objective="binary:logistic"), E.DMatrix(X, label=y), E.DMatrix(Xp)
    X, y, kw = _data(kind)
    Xp, _, _ = _data(kind, n=700, seed=1)
    dtrain = E.DMatrix(X, label=y, **kw)
    kw.pop("multi_target", None)
    return dict(BASE, **CASES[kind][0]), dtrain, E.DMatrix(Xp, **kw)


_MODELS = {}


def _model(E, kind):
    if kind not in _MODELS:
        params, dtrain, dpred = _train_data(E, kind)
        _MODELS[kind] = (params, dtrain, dpred, E.train(params, dtrain, ROUNDS))
    return _MODELS[kind]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", KINDS)
def test_ubj_model_predicts_like_its_source(E, kind, tmp_path):
    _, _, dm, bst = _model(E, kind)
    f = str(tmp_path / "m.ubj")
    bst.save_model(f)
    assert open(f, "rb").read() == bytes(bst.save_raw("ubj"))
    loaded = E.Booster(model_file=f)
    assert loaded.get_dump(dump_format="json", with_stats=True) == bst.get_dump(dump_format="json", with_stats=True)
    for rounds in (None, (2, 9)):
        _assert_same(_outputs(E, loaded, dm, rounds), _outputs(E, bst, dm, rounds), (kind, rounds))
    # the stock dialect's typed markers only; the float64 covers float32 cannot hold travel in b2.sum_hessian
    doc, typed = dec(open(f, "rb").read())
    assert all(markers == {TYPED[k]} for k, markers in typed.items()), typed
    inexact = any(not np.array_equal(t["sum_hess"].astype(np.float32).astype(np.float64), t["sum_hess"])
                  for t in bst.get_trees())
    assert ("b2.sum_hessian" in doc["learner"]["attributes"]) == inexact
    if kind in ("dart", "softprob_k3", "csr", "rank_ndcg"):   # logistic / softmax / LambdaMART hessians
        assert inexact
    # a reader that ignores the attribute gets float32 covers, which margins and leaf indices do not depend on
    doc["learner"]["attributes"].pop("b2.sum_hessian", None)
    stock = E.Booster(model_file=Enc("stock").val(doc))
    for mode in ("margin", "transformed", "leaf"):
        w = _outputs(E, bst, dm)[mode]
        assert _outputs(E, stock, dm)[mode].tobytes() == w.tobytes(), (kind, mode)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", KINDS)
def test_continuation_from_ubj_equals_continuation_from_json(E, kind, tmp_path):
    params, dtrain, _, bst = _model(E, kind)
    bst.save_model(str(tmp_path / "m.ubj"))
    bst.save_model(str(tmp_path / "m.json"))
    out = [bytes(E.train(params, dtrain, 3, xgb_model=str(tmp_path / name)).save_raw()) for name in ("m.ubj", "m.json")]
    assert out[0] == out[1]
    assert E.Booster(model_file=out[0]).num_boosted_rounds() == ROUNDS + 3


@pytest.mark.timeout(900)
def test_stock_dialect_file_predicts_like_the_json_file(E, tmp_path):
    rng = np.random.RandomState(8)
    X = rng.uniform(-3, 5, size=(2000, 3)).astype(np.float32)
    X[rng.uniform(size=X.shape) < 0.1] = np.nan
    dm = E.DMatrix(X)
    (tmp_path / "xgb.json").write_text(json.dumps(XGB_STYLE))
    (tmp_path / "xgb.ubj").write_bytes(Enc("stock").val(XGB_STYLE))
    a, b = E.Booster(model_file=str(tmp_path / "xgb.json")), E.Booster(model_file=str(tmp_path / "xgb.ubj"))
    _assert_same(_outputs(E, b, dm), _outputs(E, a, dm), "stock dialect")


@pytest.mark.timeout(1200)
def test_ray_train_save_ubj_and_predict_on_two_actors(E, tmp_path):
    if E.device_count() < 2:
        pytest.skip("needs 2 GPUs: each actor trains on its own GPU")
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    X, y, _ = _data("gbtree", n=8000)
    Xp, _, _ = _data("gbtree", n=3000, seed=2)
    bst = train(dict(BASE, objective="reg:squarederror"), RayDMatrix(X, y), ROUNDS, ray_params=RayParams(num_actors=2))
    f = str(tmp_path / "m.ubj")
    bst.save_model(f)
    loaded = E.Booster(model_file=f)
    want = bst.predict(E.DMatrix(Xp))
    assert predict(loaded, RayDMatrix(Xp), ray_params=RayParams(num_actors=2)).tobytes() == want.tobytes()
    assert predict(bst, RayDMatrix(Xp), ray_params=RayParams(num_actors=2)).tobytes() == want.tobytes()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("estimator", ["RayXGBRegressor", "RayXGBClassifier"])
def test_sklearn_estimator_ubj_round_trip(E, estimator, tmp_path):
    from xgboost_ray_b200 import RayParams
    from xgboost_ray_b200 import sklearn as S
    classify = estimator == "RayXGBClassifier"
    X, y, _ = _data("dart" if classify else "gbtree", n=4000)   # the "dart" case's label is binary
    Xp, _, _ = _data("gbtree", n=900, seed=3)
    cls = getattr(S, estimator)
    est = cls(n_estimators=10, max_depth=4, learning_rate=0.3).fit(X, y.astype(np.int32) if classify else y,
                                                                   ray_params=RayParams(num_actors=1))
    f = str(tmp_path / "m.ubj")
    est.save_model(f)
    assert open(f, "rb").read()[:2] == b"{L"
    other = cls().load_model(f)
    rp = RayParams(num_actors=1)
    assert other.predict(Xp, output_margin=True, ray_params=rp).tobytes() == \
        est.predict(Xp, output_margin=True, ray_params=rp).tobytes()
    if classify:   # a loaded classifier has no classes_: compare its probabilities
        assert other.predict_proba(Xp, ray_params=rp).tobytes() == est.predict_proba(Xp, ray_params=rp).tobytes()
    else:
        assert other.predict(Xp, ray_params=rp).tobytes() == est.predict(Xp, ray_params=rp).tobytes()
