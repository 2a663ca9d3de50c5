"""multi_strategy checks that need no device: accepted values, the refused combinations (named on both sides), and a
vector-leaf model file read back through load_model and written again unchanged."""
import json

import numpy as np
import pytest

from xgboost_ray_b200 import engine


@pytest.fixture(scope="module")
def built():
    """libb2hist.so: the engine checks the parameters (B2_CheckParams needs no device)."""
    from xgboost_ray_b200 import build
    return build.build()


@pytest.mark.parametrize("params,match", [
    ({"multi_strategy": "bogus"}, "multi_strategy='bogus'"),
    ({"multi_strategy": "multi_output_tree", "objective": "multi:softprob"}, "multi_output_tree.*multi:softprob"),
    ({"multi_strategy": "multi_output_tree", "booster": "dart"}, "multi_output_tree.*dart"),
    ({"multi_strategy": "multi_output_tree", "num_parallel_tree": 3}, "multi_output_tree.*num_parallel_tree"),
])
def test_refused(built, params, match):
    with pytest.raises(engine.XGBoostError, match=match):
        engine._check_supported(params)


@pytest.mark.parametrize("ms", [None, "one_output_per_tree", "multi_output_tree"])
def test_accepted(built, ms):
    engine._check_supported({"multi_strategy": ms, "objective": "binary:logistic"})


def vector_model(T=2):
    tree = {"base_weights": [0.1, -0.2, 0.3, 0.4, -0.5, 0.6][:3 * T], "categories": [], "categories_nodes": [],
            "categories_segments": [], "categories_sizes": [], "default_left": [1, 0, 0], "id": 0,
            "left_children": [1, -1, -1], "loss_changes": [2.5, 0.0, 0.0], "parents": [2147483647, 0, 0],
            "right_children": [2, -1, -1], "split_conditions": [0.25, 0.0, 0.0], "split_indices": [1, 0, 0],
            "split_type": [0, 0, 0], "sum_hessian": [10.0, 4.0, 6.0],
            "tree_param": {"num_deleted": "0", "num_feature": "3", "num_nodes": "3", "size_leaf_vector": str(T)}}
    return {"learner": {
        "attributes": {}, "feature_names": [], "feature_types": [],
        "gradient_booster": {"model": {"gbtree_model_param": {"num_parallel_tree": "1", "num_trees": "1"},
                                       "iteration_indptr": [0, 1], "tree_info": [0], "trees": [tree]},
                             "name": "gbtree"},
        "learner_model_param": {"base_score": "0.5", "boost_from_average": "1", "num_class": "0", "num_feature": "3",
                                "num_target": str(T)},
        "objective": {"name": "reg:squarederror", "reg_loss_param": {"scale_pos_weight": "1"}}},
        "version": [2, 0, 3]}


def test_vector_model_file_round_trip():
    raw = json.dumps(vector_model()).encode()
    b = engine.Booster()
    b.load_model(bytearray(raw))
    assert b.is_vector_leaf and b.params["multi_strategy"] == "multi_output_tree" and b.num_class == 2
    t = b.get_trees()[0]
    assert t["leaf_vector"].shape == (3, 2)
    assert np.array_equal(t["leaf_vector"], np.float32([[0.1, -0.2], [0.3, 0.4], [-0.5, 0.6]]))
    assert "1:leaf=[0.300000012,0.400000006]" in b.get_dump()[0]
    out = json.loads(bytes(b.save_raw()))
    tree = out["learner"]["gradient_booster"]["model"]["trees"][0]
    assert tree["tree_param"]["size_leaf_vector"] == "2"
    assert tree["base_weights"] == [float(np.float32(x)) for x in vector_model()["learner"]["gradient_booster"]["model"]
                                    ["trees"][0]["base_weights"]]
    assert tree["split_conditions"] == [0.25, 0.0, 0.0]
    assert out["learner"]["gradient_booster"]["model"]["tree_info"] == [0]
    assert out["learner"]["gradient_booster"]["model"]["iteration_indptr"] == [0, 1]
    assert json.loads(b.save_config())["learner"]["learner_train_param"]["multi_strategy"] == "multi_output_tree"
    assert b.num_boosted_rounds() == 1


def test_leaf_vector_size_must_match_targets():
    m = vector_model()
    m["learner"]["learner_model_param"]["num_target"] = "3"
    with pytest.raises(engine.XGBoostError, match="size 2 for 3 targets"):
        engine.Booster().load_model(bytearray(json.dumps(m).encode()))
