"""UBJSON model files (DESIGN.md 2 item 25) without a GPU: save_raw("ubj"), save_model("*.ubj") and load_model of either
format.

The encoder and decoder here are written from the UBJSON draft 12 spec with `struct` and share no code with
xgboost_ray_b200/ubjson.py: the test decoder checks what the engine writes against json.loads of its JSON file, and the
test encoder writes every model in several legal forms that must all load to the same model."""
import base64
import json
import os
import pathlib
import pickle
import re
import struct

import jsonschema
import numpy as np
import pytest

from tests.model_files import xgb_model_file
from tests.model_schema import MODEL
from tests.test_model_json import XGB_STYLE, _booster_from_golden
from tests.test_model_slicing import CASES as SLICING_CASES
from xgboost_ray_b200 import engine as E

# the typed tree arrays of xgboost 2.x's dialect and their element markers
TYPED = {"split_conditions": "d", "base_weights": "d", "loss_changes": "d", "sum_hessian": "d", "weight_drop": "d",
         "left_children": "l", "right_children": "l", "parents": "l", "split_indices": "l", "categories": "l",
         "categories_nodes": "l", "default_left": "U", "split_type": "U", "categories_segments": "L",
         "categories_sizes": "L"}
FMT = {"i": ">b", "U": ">B", "I": ">h", "l": ">i", "L": ">q", "d": ">f", "D": ">d"}


# ----------------------------------------------------------------------------- test decoder
class Dec:
    """Recursive draft-12 reader; records the marker of every typed array under its key."""

    def __init__(self, b):
        self.b, self.p, self.typed = b, 0, {}

    def byte(self):
        c = chr(self.b[self.p])
        self.p += 1
        return c

    def num(self, m):
        v = struct.unpack_from(FMT[m], self.b, self.p)[0]
        self.p += struct.calcsize(FMT[m])
        return v

    def int_(self):
        m = self.byte()
        assert m in "iUIlL", m
        return self.num(m)

    def str_(self):
        n = self.int_()
        s = self.b[self.p:self.p + n].decode("utf-8")
        self.p += n
        return s

    def val(self, m=None, key=None):
        m = m or self.byte()
        if m in FMT:
            return self.num(m)
        if m == "S":
            return self.str_()
        if m in "TFZ":
            return {"T": True, "F": False, "Z": None}[m]
        if m in "[{":
            t = n = None
            if chr(self.b[self.p]) == "$":
                self.p += 1
                t = self.byte()
            if chr(self.b[self.p]) == "#":
                self.p += 1
                n = self.int_()
            if t is not None and key is not None:
                self.typed.setdefault(key, set()).add(t)
            out = {} if m == "{" else []
            while True:
                if n is None and chr(self.b[self.p]) in "]}":
                    self.p += 1
                    return out
                if n is not None and len(out) == n:
                    return out
                if m == "{":
                    k = self.str_()
                    out[k] = self.val(t, k)
                else:
                    out.append(self.val(t, key))
        raise AssertionError("marker %r at %d" % (m, self.p - 1))


def dec(b):
    d = Dec(bytes(b))
    v = d.val()
    assert d.p == len(d.b)
    return v, d.typed


# ----------------------------------------------------------------------------- test encoder
class Enc:
    """Draft-12 writer of a JSON document in one of several legal forms."""

    def __init__(self, form, width="L"):
        self.form, self.width = form, width

    def int_(self, v):
        order = "iUIlL"["iUIlL".index(self.width):] if self.form == "widths" else "L"
        for m in order:
            try:
                return m.encode() + struct.pack(FMT[m], v)
            except struct.error:
                pass
        raise AssertionError(v)

    def str_(self, s):
        b = s.encode("utf-8")
        return self.int_(len(b)) + b

    def flt(self, v):
        if self.form == "D" or not (v != v or float(np.float32(v)) == v):   # "D": every float as float64
            return b"D" + struct.pack(">d", v)
        return b"d" + struct.pack(">f", v)

    def val(self, v, key=None):
        if self.form == "H" and isinstance(v, (int, float)) and not isinstance(v, bool):
            return b"H" + self.str_(repr(v))
        if isinstance(v, bool):
            return b"T" if v else b"F"
        if v is None:
            return b"Z"
        if isinstance(v, int):
            return self.int_(v)
        if isinstance(v, float):
            return self.flt(v)
        if isinstance(v, str):
            return b"S" + self.str_(v)
        noop = b"N" if self.form == "noop" else b""
        if isinstance(v, dict):
            body = b"".join(noop + self.str_(k) + noop + self.val(x, k) for k, x in v.items())
            if self.form == "counted":
                return b"{#" + self.int_(len(v)) + body
            return b"{" + body + noop + b"}"
        if key in TYPED and self.form in ("stock", "widths", "D"):
            t = TYPED[key]
            if t == "d":
                t = "D" if self.form == "D" or any(float(np.float32(x)) != x for x in v) else "d"
                data = b"".join(struct.pack(FMT[t], float(x)) for x in v)
            else:
                if self.form == "widths":   # the narrowest typed integer at or above `width` that holds the array
                    t = next(m for m in "iUIlL"["iUIlL".index(self.width):]
                             if all(_fits(m, x) for x in v))
                data = b"".join(struct.pack(FMT[t], x) for x in v)
            return b"[$" + t.encode() + b"#" + self.int_(len(v)) + data
        body = b"".join(noop + self.val(x) for x in v)
        if self.form == "counted":
            return b"[#" + self.int_(len(v)) + body
        return b"[" + body + noop + b"]"


def _fits(m, x):
    try:
        struct.pack(FMT[m], x)
        return True
    except struct.error:
        return False


FORMS = [("stock", "L"), ("countless", "L"), ("counted", "L"), ("D", "L"), ("noop", "L"), ("H", "L")] + \
        [("widths", w) for w in "iUIlL"]


# ----------------------------------------------------------------------------- the models
def _non_ascii():
    d = json.loads(xgb_model_file(4, attrs={"note": "Größe °C"}).decode())
    d["learner"]["feature_names"] = ["größe", "温度", "f_ü", "имя"]
    return json.dumps(d).encode()


def _float64_covers():
    """A logistic model whose hessian sums float32 cannot hold, as this engine's float64 covers usually are."""
    d = json.loads(xgb_model_file(4, objective="binary:logistic").decode())
    for i, t in enumerate(d["learner"]["gradient_booster"]["model"]["trees"]):
        t["sum_hessian"] = [2.3 + i / 7, 1.1 + i / 7, 1.2]
    return json.dumps(d).encode()


def _models():
    out = {"xgb_style": json.dumps(XGB_STYLE).encode(), "gbtree": xgb_model_file(5)}
    out.update({k: xgb_model_file(5, **v) for k, v in SLICING_CASES.items()})
    out["interaction_constraints"] = xgb_model_file(
        5, attrs={"b2.params": json.dumps({"interaction_constraints": "[[0, 1], [2, 3]]"})})
    out["non_ascii_names"] = _non_ascii()
    out["float64_covers"] = _float64_covers()
    for g in ("breast_cancer_logistic.json", "synthetic_categorical_softprob.json"):
        out[g] = bytes(_booster_from_golden(g)[0].save_raw())
    return out


MODELS = _models()


def _load(raw):
    return E.Booster(model_file=bytearray(raw))


def _same(a, b, path="$"):
    """Equal documents: same keys in the same order, same types, floats equal as float32 bits."""
    assert type(a) is type(b), (path, type(a), type(b))
    if isinstance(a, dict):
        assert list(a) == list(b), path
        for k in a:
            _same(a[k], b[k], path + "." + k)
    elif isinstance(a, list):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, "%s[%d]" % (path, i))
    elif isinstance(a, float):
        assert np.float32(a).tobytes() == np.float32(b).tobytes(), (path, a, b)
    else:
        assert a == b, (path, a, b)


@pytest.mark.parametrize("name", list(MODELS))
def test_round_trip_through_the_engine(name):
    b = _load(MODELS[name])
    j, u = bytes(b.save_raw()), bytes(b.save_raw("ubj"))
    via_json = bytes(_load(j).save_raw())
    b2 = _load(u)
    assert bytes(b2.save_raw()) == via_json
    assert bytes(b2.save_raw("ubj")) == bytes(_load(j).save_raw("ubj"))
    if name != "quantile_3_alphas":   # a loaded quantile model writes its alphas as the file's float32 text
        assert via_json == j and bytes(b2.save_raw("ubj")) == u
    u2 = bytes(b2.save_raw("ubj"))
    assert bytes(_load(u2).save_raw("ubj")) == u2
    assert b2.get_dump(dump_format="json", with_stats=True) == b.get_dump(dump_format="json", with_stats=True)
    assert b2.get_tree_weights().tobytes() == b.get_tree_weights().tobytes()


@pytest.mark.parametrize("name", list(MODELS))
def test_encoder_checked_by_an_independent_decoder(name):
    b = _load(MODELS[name])
    j = json.loads(bytes(b.save_raw()).decode())
    doc, typed = dec(b.save_raw("ubj"))
    covers = json.loads(doc["learner"]["attributes"].pop("b2.sum_hessian", "[]"))
    _same(doc, j)
    gb = j["learner"]["gradient_booster"]
    trees = (gb["gbtree"] if gb["name"] == "dart" else gb)["model"]["trees"]
    inexact = [i for i, t in enumerate(trees) if any(float(np.float32(x)) != x for x in t["sum_hessian"])]
    assert [i for i, _ in covers] == inexact and (name == "float64_covers") == bool(inexact)
    for i, b64 in covers:   # the exact covers: little-endian float64
        assert np.frombuffer(base64.b64decode(b64), "<f8").tolist() == trees[i]["sum_hessian"]
    gb = doc["learner"]["gradient_booster"]
    want = set(TYPED) - ({"weight_drop"} if gb["name"] != "dart" else set())
    assert set(typed) == want
    for k, markers in typed.items():
        assert markers == {TYPED[k]}, k
    if gb["name"] == "gbtree" and doc["learner"]["objective"]["name"] in ("reg:squarederror", "binary:logistic",
                                                                          "multi:softprob", "multi:softmax"):
        jsonschema.validate(doc, MODEL)
    raw = bytes(b.save_raw("ubj"))
    assert raw[:1] == b"{" and raw[1:2] == b"L"   # keys: an int64 length, then the bytes


def test_feature_names_are_utf8():
    b = _load(MODELS["non_ascii_names"])
    raw = bytes(b.save_raw("ubj"))
    assert "温度".encode("utf-8") in raw and "Größe °C".encode("utf-8") in raw
    assert _load(raw).feature_names == ["größe", "温度", "f_ü", "имя"]


def test_float64_covers_travel_in_an_attribute():
    b = _load(MODELS["float64_covers"])
    raw = bytes(b.save_raw("ubj"))
    doc, typed = dec(raw)
    assert typed["sum_hessian"] == {"d"}                     # the stock dialect's float32 array
    attrs = doc["learner"]["attributes"]
    assert "b2.sum_hessian" in attrs and "b2.sum_hessian" not in json.loads(bytes(b.save_raw()).decode())["learner"]["attributes"]
    b2 = _load(raw)
    for t, u in zip(b._trees, b2._trees):
        assert u["sum_hess"].dtype == np.float64 and u["sum_hess"].tobytes() == t["sum_hess"].tobytes()
    assert bytes(b2.save_raw()) == bytes(b.save_raw()) and "b2.sum_hessian" not in b2.attributes()
    # what a reader that ignores the attribute sees: the float32 covers
    del attrs["b2.sum_hessian"]
    stock = _load(Enc("stock").val(doc))
    for t, u in zip(b._trees, stock._trees):
        assert u["sum_hess"].tobytes() == t["sum_hess"].astype(np.float32).astype(np.float64).tobytes()
    assert bytes(stock.save_raw("ubj")) == bytes(Enc("stock").val(doc))


def test_attribute_covers_yield_to_rewritten_trees():
    """Covers in b2.sum_hessian that do not round to the file's sum_hessian (the trees were rewritten by a tool that
    kept the attribute) are not used; a malformed attribute is refused."""
    b = _load(MODELS["float64_covers"])
    doc, _ = dec(b.save_raw("ubj"))
    doc["learner"]["gradient_booster"]["model"]["trees"][0]["sum_hessian"] = [5.0, 2.0, 3.0]
    got = _load(Enc("stock").val(doc))
    assert got._trees[0]["sum_hess"].tolist() == [5.0, 2.0, 3.0]
    assert got._trees[1]["sum_hess"].tobytes() == b._trees[1]["sum_hess"].tobytes()
    for bad in ("[[0,\"not base64!\"]]", "{", "[[0]]"):
        doc["learner"]["attributes"]["b2.sum_hessian"] = bad
        with pytest.raises(E.XGBoostError, match="b2.sum_hessian is malformed"):
            _load(Enc("stock").val(doc))


def test_typed_float_arrays_never_round():
    from xgboost_ray_b200 import ubjson
    assert ubjson.dumps({"sum_hessian": [0.5, 2.0]}) == b"{L" + struct.pack(">q", 11) + b"sum_hessian[$d#L" + \
        struct.pack(">q", 2) + struct.pack(">ff", 0.5, 2.0) + b"}"
    with pytest.raises(E.XGBoostError, match="float32 cannot hold exactly"):
        ubjson.dumps({"sum_hessian": [0.1]})


@pytest.mark.parametrize("form,width", FORMS)
@pytest.mark.parametrize("name", list(MODELS))
def test_decoder_reads_every_form(name, form, width):
    j = json.loads(MODELS[name].decode())
    want = bytes(_load(MODELS[name]).save_raw())
    raw = Enc(form, width).val(j)
    assert bytes(_load(raw).save_raw()) == want


def test_decoder_values():
    from xgboost_ray_b200 import ubjson
    for m, dt in (("i", np.int8), ("U", np.uint8), ("I", np.int16), ("l", np.int32), ("L", np.int64),
                  ("d", np.float32), ("D", np.float64)):
        vals = np.array([0, 1, 100, 7, 0], dtype=dt)
        a = ubjson.loads(b"[$" + m.encode() + b"#i\x05" + vals.astype(np.dtype(dt).newbyteorder(">")).tobytes())
        assert isinstance(a, np.ndarray) and a.dtype == np.dtype(dt) and a.dtype.isnative and np.array_equal(a, vals)
    nan_inf = b"[#U\x03" + b"d" + struct.pack(">f", float("nan")) + b"D" + struct.pack(">d", float("inf")) + \
        b"d" + struct.pack(">f", float("-inf"))
    v = ubjson.loads(nan_inf)
    assert np.isnan(v[0]) and v[1] == float("inf") and v[2] == float("-inf")
    assert ubjson.loads(b"[$T#i\x03") == [True] * 3
    assert ubjson.loads(b"[$Z#U\x02") == [None, None]
    assert ubjson.loads(b"{$S#i\x02i\x01ai\x01xU\x02bci\x00") == {"a": "x", "bc": ""}
    assert ubjson.loads(b"[$[#i\x02#i\x01T]") == [[True], []]
    assert ubjson.loads(b"[CaHi\x041e+2Hi\x02-7N]") == ["a", 100.0, -7]
    deep = 50000
    v = ubjson.loads(b"[" * deep + b"i\x05" + b"]" * deep)
    for _ in range(deep):
        v = v[0] if isinstance(v, list) else v
    assert v == 5


def _offset(e):
    m = re.search(r"at byte offset (\d+)", str(e))
    assert m, str(e)
    return int(m.group(1))


def test_truncated_at_every_byte():
    raw = bytes(_load(MODELS["xgb_style"]).save_raw("ubj"))
    for n in range(len(raw)):
        with pytest.raises(E.XGBoostError) as e:
            _load(raw[:n])
        if n >= 2:
            assert re.search("truncated|runs past the end", str(e.value)) and _offset(e.value) <= n, n
        else:
            assert "not a JSON or UBJSON model" in str(e.value)


KEY = b"i\x01a"
BAD = [
    (b"{" + KEY + b"X}", 4, "unknown marker 'X'"),
    (b"{" + KEY + b"[#i\xfe]}", 6, "negative count -2"),
    (b"{" + KEY + b"Si\xff}", 5, "negative string length -1"),
    (b"{" + KEY + b"[$d#i\x03" + b"\x00" * 8 + b"}", 8, "count 3 of 'd' values runs past the end"),
    (b"{" + KEY + b"[#I\x01\x00Z]}", 6, "count 256 runs past the end"),
    (b"{" + KEY + b"Si\x09abc}", 7, "truncated"),
    (b"{" + KEY + b"Z}Z", 6, "1 trailing bytes"),
    (b"{" + KEY + b"Z}" + b"\x00" * 5, 6, "5 trailing bytes"),
    (b"{" + KEY + b"ZSi\x01bZ}", 5, "object key must be a string"),
    (b"{" + KEY + b"Zdi\x01bZ}", 5, "object key must be a string"),
    (b"{" + KEY + b"[$d]}", 7, "'$' type 'd' without a '#' count"),
    (b"{" + KEY + b"[$Q#i\x01}", 6, "'Q' is not a value type"),
    (b"{" + KEY + b"Si\x02\xff\xfe}", 7, "not UTF-8"),
    (b"{" + KEY + b"Hi\x021x}", 4, "not a JSON number"),
    (b"{" + KEY + b"[$T#L\x7f" + b"\xff" * 7 + b"}", 8, "exceeds the limit of 16777216"),
    (b"{" + KEY + b"[$Z#l\x01\x00\x00\x01]}", 8, "exceeds the limit"),
    (b"{" + KEY + b"{$Z#L\x7f" + b"\xff" * 7 + b"}", 8, "runs past the end"),
]


@pytest.mark.parametrize("raw,offset,reason", BAD)
def test_malformed_input_names_its_offset(raw, offset, reason):
    with pytest.raises(E.XGBoostError, match=re.escape(reason)) as e:
        _load(raw)
    assert _offset(e.value) == offset


@pytest.mark.parametrize("raw", [b"", b"\x00\x01\x02", b"binf\x00", b"[1, 2]", b"{'a': 1}", b"  {", b"{X",
                                 b"\xef\xbb\xbf{}"])
def test_neither_format(raw):
    with pytest.raises(E.XGBoostError, match="not a JSON or UBJSON model; the deprecated binary format is not supported"):
        _load(raw)


@pytest.mark.parametrize("fmt,match", [("deprecated", "old binary model format, is not supported"),
                                       ("foo", "raw_format='foo' is not supported"), ("UBJ", "supported: json, ubj")])
def test_unsupported_raw_format(fmt, match):
    with pytest.raises(E.XGBoostError, match=match):
        _load(MODELS["gbtree"]).save_raw(fmt)


def test_leading_whitespace_before_either_format():
    b = _load(MODELS["gbtree"])
    want = bytes(b.save_raw())
    for raw in (b" \n" + want, b"\t" + bytes(b.save_raw("ubj"))):
        assert bytes(_load(raw).save_raw()) == want


@pytest.mark.parametrize("name,ubj", [("m.ubj", True), ("m.json", False), ("m.model", False), ("m", False),
                                      ("m.ubj.json", False), ("m.json.ubj", True),
                                      ("m.UBJ", True), ("m.Ubj", True)])
@pytest.mark.parametrize("as_path", [False, True])
def test_save_model_format_follows_the_suffix(tmp_path, name, ubj, as_path):
    b = _load(MODELS["dart"])
    f = tmp_path / name
    b.save_model(f if as_path else str(f))
    raw = f.read_bytes()
    assert raw == bytes(b.save_raw("ubj" if ubj else "json"))
    assert bytes(E.Booster(model_file=f if as_path else str(f)).save_raw()) == bytes(b.save_raw())


def test_load_model_reads_the_content_not_the_name(tmp_path):
    b = _load(MODELS["softprob_k20"])
    want = bytes(b.save_raw())
    for name, fmt in (("a.json", "ubj"), ("b.ubj", "json"), ("c", "ubj"), ("d.bin", "json")):
        f = tmp_path / name
        f.write_bytes(bytes(b.save_raw(fmt)))
        c = E.Booster()
        c.load_model(str(f))
        assert bytes(c.save_raw()) == want
        assert bytes(E.Booster(model_file=pathlib.Path(f)).save_raw()) == want
    assert bytes(_load(bytes(b.save_raw("ubj"))).save_raw()) == want   # bytes as well as bytearray


def test_sklearn_estimators_save_and_load_ubj(tmp_path):
    from xgboost_ray_b200.sklearn import RayXGBClassifier, RayXGBRegressor
    for cls, name in ((RayXGBRegressor, "gbtree"), (RayXGBClassifier, "xgb_style")):
        est = cls()
        est._Booster = _load(MODELS[name])
        f = str(tmp_path / (name + ".ubj"))
        est.save_model(f)
        assert open(f, "rb").read() == bytes(est.get_booster().save_raw("ubj"))
        other = cls().load_model(f)
        assert bytes(other.get_booster().save_raw()) == bytes(est.get_booster().save_raw())
        assert other.n_features_in_ == est.get_booster().n_features


@pytest.mark.parametrize("name", ["gbtree", "dart", "quantile_3_alphas", "non_ascii_names", "breast_cancer_logistic.json"])
def test_json_and_pickle_bytes_are_unchanged(name):
    b = _load(MODELS[name])
    parent = json.dumps(b._model_dict(), allow_nan=False).encode()   # what save_raw() wrote before it took a format
    assert bytes(b.save_raw()) == parent and bytes(b.save_raw("json")) == parent
    state = b.__getstate__()
    assert state["raw"] == parent and set(state) == {"raw", "best_iteration", "best_score", "cuts"}
    assert bytes(pickle.loads(pickle.dumps(b)).save_raw()) == bytes(_load(parent).save_raw())

