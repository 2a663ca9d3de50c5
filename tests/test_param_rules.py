"""Every refusal of the engine's parameter parser (params.cu parse_params / set_targets), without a device: the Python
check (_check_supported) and a raw B2_CheckParams call on the same text fail with the same message."""
import re

import pytest

from xgboost_ray_b200 import engine as E


@pytest.fixture(scope="module")
def built():
    from xgboost_ray_b200 import build
    return build.build()


def raw_check(text):
    """(return code, message) of B2_CheckParams on `text`."""
    lib = E.lib()
    rc = lib.B2_CheckParams(text.encode())
    return rc, lib.B2_GetLastError().decode() if rc else None


UPD = {"process_type": "update", "updater": "refresh"}
VEC = {"multi_strategy": "multi_output_tree"}

REFUSED = [
    # set_targets: the rules that need the label width (num_target)
    ({"num_target": 0}, r"num_target must be in \[1, 4096\], got 0"),
    ({"num_target": 4097}, r"num_target must be in \[1, 4096\], got 4097"),
    ({"objective": "count:poisson", "num_target": 2}, "objective 'count:poisson' does not support a label with 2 columns"),
    ({"num_class": 3, "num_target": 2}, "num_class must not be set with a label of 2 columns"),
    (dict(VEC, num_target=65), "multi_strategy='multi_output_tree' supports at most 64 targets, the label has 65 columns"),
    (dict(UPD, num_target=3, **VEC), "process_type='update' is not supported with multi_strategy='multi_output_tree'"),
    # parse_params: one value at a time
    ({"objective": "reg:absoluteerror"}, "unsupported objective 'reg:absoluteerror'"),
    ({"objective": "survival:cox"},
     "^" + re.escape("unsupported objective 'survival:cox' (supported: reg:squarederror, reg:logistic, binary:logistic, "
                     "binary:logitraw, reg:squaredlogerror, reg:pseudohubererror, count:poisson, reg:gamma, reg:tweedie, "
                     "survival:aft, rank:pairwise, rank:ndcg, rank:map, reg:quantileerror, multi:softprob, "
                     "multi:softmax)") + "$"),
    ({"aft_loss_distribution": "cauchy"}, "aft_loss_distribution must be normal, logistic or extreme, got 'cauchy'"),
    ({"lambdarank_pair_method": "mean"}, "lambdarank_pair_method='mean' is not supported"),
    ({"lambdarank_num_pair_per_sample": 0}, "lambdarank_num_pair_per_sample must be an integer >= 1, got '0'"),
    ({"ndcg_exp_gain": "maybe"}, "ndcg_exp_gain must be a boolean, got 'maybe'"),
    ({"lambdarank_unbiased": True}, "lambdarank_unbiased=true is not supported"),
    ({"multi_strategy": "bogus"}, r"multi_strategy='bogus' is not supported \(supported: one_output_per_tree, "),
    ({"booster": "gblinear"}, r"booster='gblinear' is not supported \(supported: gbtree, dart\)"),
    ({"process_type": "sideways"}, r"process_type='sideways' is not supported \(supported: 'default', 'update'\)"),
    (dict(UPD, refresh_leaf=2), "refresh_leaf must be 0 or 1, got '2'"),
    ({"updater": "prune"}, "updater='prune' is not supported"),
    (dict(UPD, updater="refresh,prune"), "updater='refresh,prune' is not supported"),
    ({"booster": "dart", "sample_type": "x"}, "sample_type must be uniform or weighted, got 'x'"),
    ({"booster": "dart", "normalize_type": "x"}, "normalize_type must be tree or forest, got 'x'"),
    ({"booster": "dart", "one_drop": 2}, "one_drop must be 0 or 1, got '2'"),
    ({"booster": "dart", "rate_drop": 1.5}, r"rate_drop must be a number in \[0, 1\], got '1.5'"),
    ({"booster": "dart", "skip_drop": -0.5}, r"skip_drop must be a number in \[0, 1\], got '-0.5'"),
    # parse_params: parameters that do not go together
    ({"objective": "rank:ndcg", "num_class": 3}, "rank:ndcg has one output per row: num_class must be 1, got 3"),
    ({"objective": "reg:quantileerror", "num_class": 3},
     r"reg:quantileerror has one output per quantile_alpha: num_class must not be set \(got 3\)"),
    ({"objective": "reg:quantileerror", "booster": "dart"}, "reg:quantileerror is not supported with booster='dart'"),
    ({"objective": "reg:quantileerror", "num_parallel_tree": 2}, r"reg:quantileerror needs num_parallel_tree = 1 \(got 2\)"),
    (dict(VEC, objective="multi:softmax", num_class=3),
     "multi_strategy='multi_output_tree' is not supported with objective='multi:softmax': vector-leaf trees take the "
     "multi-target objectives"),
    # one target: refused whatever the label width (the engine used to refuse these only with num_target > 1)
    (dict(VEC, booster="dart"), "multi_strategy='multi_output_tree' is not supported with booster='dart'"),
    (dict(VEC, num_parallel_tree=3), r"multi_strategy='multi_output_tree' needs num_parallel_tree = 1 \(got 3\)"),
    ({"objective": "multi:softprob"}, "multi:softprob needs num_class >= 2"),
    ({"process_type": "update"}, "process_type='update' needs updater='refresh', got updater=''"),
    (dict(UPD, updater="grow_gpu_hist"), "process_type='update' needs updater='refresh', got updater='grow_gpu_hist'"),
    (dict(UPD, booster="dart"), "process_type='update' is not supported with booster='dart'"),
    (dict(UPD, objective="reg:quantileerror"),
     "process_type='update' is not supported with objective='reg:quantileerror': its leaf values are residual quantiles"),
    ({"updater": "refresh"}, "updater='refresh' needs process_type='update'"),
    # parse_params: ranges
    ({"max_depth": 0}, r"max_depth must be in \[1, 16\], got 0"),
    ({"max_depth": 17}, r"max_depth must be in \[1, 16\], got 17"),
    ({"num_parallel_tree": 0}, r"num_parallel_tree must be in \[1, 4096\], got 0"),
    ({"hist_qbits": 7}, r"hist_qbits must be in \[8, 24\], got 7"),
    ({"colsample_bynode": 0}, r"subsample / colsample_\* must be in \(0, 1\], got 0"),
    ({"subsample": 1.5}, r"subsample / colsample_\* must be in \(0, 1\], got 1.5"),
    ({"max_cat_to_onehot": 0}, "max_cat_to_onehot must be >= 1, got 0"),
    ({"max_cat_threshold": 0}, "max_cat_threshold must be >= 1, got 0"),
    ({"objective": "count:poisson", "max_delta_step": -1}, "max_delta_step must be >= 0 for count:poisson, got -1"),
    ({"objective": "reg:pseudohubererror", "huber_slope": 0}, "huber_slope must be > 0 for reg:pseudohubererror, got 0"),
    ({"objective": "reg:tweedie", "tweedie_variance_power": 2}, r"tweedie_variance_power must be in \[1, 2\), got 2"),
    ({"aft_loss_distribution_scale": 0}, "aft_loss_distribution_scale must be finite and > 0, got 0"),
    ({"objective": "reg:logistic", "base_score": 1.5}, r"base_score must be in \(0, 1\) for reg:logistic, got 1.5"),
    ({"objective": "reg:gamma", "base_score": 0}, "base_score must be > 0 for reg:gamma, got 0"),
]


def _ids(table):
    return ["-".join("%s=%s" % kv for kv in params.items()) for params, _ in table]


@pytest.mark.parametrize("params,match", REFUSED, ids=_ids(REFUSED))
def test_refusal(built, params, match):
    with pytest.raises(E.XGBoostError, match=match) as e:
        E._check_supported(params)
    text = "\n".join("%s=%s" % kv for kv in params.items())
    assert raw_check(text) == (-1, str(e.value))


@pytest.mark.parametrize("text,match", [
    # engine text that Python writes itself from the user's value (and refuses in its own words first)
    ("interaction_constraints=0,1;2,x", "interaction_constraints: 'x' is not a feature index"),
    ("quantile_alpha=0.5,1.5", r"quantile_alpha: '1.5' is not a number in \(0, 1\)"),
])
def test_refusal_of_engine_text(built, text, match):
    rc, msg = raw_check(text)
    assert rc == -1 and re.search(match, msg), msg


@pytest.mark.parametrize("params", [
    {}, {"objective": "multi:softprob", "num_class": 3}, dict(VEC, num_target=64), dict(VEC, objective="binary:logistic"),
    dict(UPD, refresh_leaf="false"), {"updater": "grow_quantile_histmaker"}, {"booster": "dart", "rate_drop": 0.1},
    {"objective": "reg:quantileerror", "quantile_alpha": [0.1, 0.9]}, {"objective": "rank:map"},
    {"booster": "gbtree", "sample_type": "x"},   # DART's parameters are ignored by gbtree, like xgboost
    # every other accepted objective name
    *({"objective": o} for o in ("reg:squarederror", "reg:linear", "reg:logistic", "binary:logistic", "binary:logitraw",
                                 "reg:squaredlogerror", "reg:pseudohubererror", "count:poisson", "reg:gamma",
                                 "reg:tweedie", "survival:aft", "rank:pairwise", "rank:ndcg")),
    {"objective": "multi:softmax", "num_class": 3},
])
def test_accepted(built, params):
    E._check_supported(params)
    assert raw_check(E._engine_text(params).decode()) == (0, None)
