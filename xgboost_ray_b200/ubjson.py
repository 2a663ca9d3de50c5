"""UBJSON (Universal Binary JSON, draft 12): xgboost's binary model format (DESIGN.md §2 item 25).

`loads` reads any conforming document.  Typed numeric arrays (`[$d#...`, `[$l#...`, ...) become NumPy arrays in native
byte order, read in one call each, so a large model never goes through per-element Python code.  Malformed input raises
XGBoostError naming the byte offset.

`dumps` writes the dialect xgboost 2.x writes for a model: keys as a length and the bytes, strings `S`, integers `L`,
floats `d`, booleans `T` / `F`, untyped `{ }` and `[ ]` containers, and the tree arrays of XGBOOST_TYPED as typed arrays
with an `L` count.  The encoder never rounds: a float array of XGBOOST_TYPED must hold float32 values (the caller
rounds, and keeps what float32 cannot hold elsewhere), and a scalar float that float32 cannot hold is written as `D`.
"""
import re
import struct

import numpy as np

from xgboost_ray_b200.engine import XGBoostError

# element type of each typed array xgboost 2.x writes in a model (by object key); every other array is untyped
XGBOOST_TYPED = {
    "split_conditions": "d", "base_weights": "d", "loss_changes": "d", "sum_hessian": "d", "weight_drop": "d",
    "left_children": "l", "right_children": "l", "parents": "l", "split_indices": "l", "categories": "l",
    "categories_nodes": "l",
    "default_left": "U", "split_type": "U",
    "categories_segments": "L", "categories_sizes": "L",
}

_STRUCT = {"i": ">b", "U": ">B", "I": ">h", "l": ">i", "L": ">q", "d": ">f", "D": ">d"}
_INTS = "iUIlL"
_NATIVE = {m: np.dtype(f[1:]) for m, f in _STRUCT.items()}   # native byte order
_BIG = {m: np.dtype(f) for m, f in _STRUCT.items()}
_VALUE_MARKERS = set("ZTFiUIlLdDHCS[{")
_HNUM = re.compile(rb"-?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?\Z")
# `[$Z#n`, `[$T#n` and `[$F#n` take no bytes per element, so the buffer cannot bound n: each element still costs a
# Python object, and a larger count is refused rather than exhausting memory
MAX_EMPTY_ELEMENTS = 1 << 24


class _Frame:
    """An open container: its contents so far, the key awaiting its value (objects), the entries still to come
    (`#` count, or None until the closing marker) and the element type (`$`, or None)."""
    __slots__ = ("out", "obj", "left", "typ", "key")

    def __init__(self, obj, left, typ):
        self.out = {} if obj else []
        self.obj, self.left, self.typ, self.key = obj, left, typ, None

    def put(self, v):
        if self.obj:
            self.out[self.key] = v
        else:
            self.out.append(v)
        if self.left is not None:
            self.left -= 1


class _Reader:
    def __init__(self, buf, pos):
        self.buf, self.pos, self.end = buf, pos, len(buf)

    def fail(self, what, at=None):
        raise XGBoostError("UBJSON: %s at byte offset %d" % (what, self.pos if at is None else at))

    def take(self, n, what):
        """Offset of the next n bytes, which must lie inside the buffer."""
        if n > self.end - self.pos:
            self.fail("truncated: %s of %d bytes runs past the end (%d bytes left)" % (what, n, self.end - self.pos))
        p = self.pos
        self.pos += n
        return p

    def peek(self, what):
        if self.pos >= self.end:
            self.fail("truncated: expected %s" % what)
        return chr(self.buf[self.pos])

    def marker(self, what="a value"):
        """The next marker, after any no-op `N`s."""
        while self.peek(what) == "N":
            self.pos += 1
        self.pos += 1
        return chr(self.buf[self.pos - 1])

    def number(self, m):
        return struct.unpack_from(_STRUCT[m], self.buf, self.take(_BIG[m].itemsize, "%r number" % m))[0]

    def length(self, what):
        at = self.pos
        m = self.marker(what)
        if m not in _INTS:
            self.fail("%s must be an integer (i U I l L), found marker %r" % (what, m), at)
        n = self.number(m)
        if n < 0:
            self.fail("negative %s %d" % (what, n), at)
        return n

    def text(self, what):
        n = self.length(what + " length")
        p = self.take(n, what)
        try:
            return bytes(self.buf[p:p + n]).decode("utf-8")
        except UnicodeDecodeError as e:
            self.fail("%s is not UTF-8 (%s)" % (what, e.reason), p + e.start)

    def key(self):
        at = self.pos
        if self.peek("an object key") not in _INTS + "N":
            self.fail("object key must be a string (a length, then UTF-8 bytes), found marker %r"
                      % self.peek("an object key"), at)
        return self.text("object key")

    def scalar(self, m, at):
        if m == "Z":
            return None
        if m == "T":
            return True
        if m == "F":
            return False
        if m in _STRUCT:
            return self.number(m)
        if m == "S":
            return self.text("string")
        if m == "C":
            c = self.buf[self.take(1, "char")]
            if c > 127:
                self.fail("char %d is not ASCII" % c, self.pos - 1)
            return chr(c)
        if m == "H":
            s = self.text("high-precision number").encode()
            if not _HNUM.match(s):
                self.fail("high-precision number %r is not a JSON number" % s.decode(), at)
            return float(s) if any(c in s for c in b".eE") else int(s)
        self.fail("unknown marker %r" % m, at)

    def open(self, m):
        """A container's header (`$` type, `#` count): a typed numeric array is read whole, anything else opens."""
        typ = left = None
        if self.peek("container contents") == "$":
            self.pos += 1
            at = self.pos
            typ = chr(self.buf[self.take(1, "'$' type")])
            if typ not in _VALUE_MARKERS:
                self.fail("%r is not a value type for '$'" % typ, at)
            if self.peek("'#' count") != "#":
                self.fail("'$' type %r without a '#' count" % typ)
        if self.peek("container contents") == "#":
            self.pos += 1
            at = self.pos
            left = self.length("count")
            if m == "[" and typ in _STRUCT:
                size = _BIG[typ].itemsize
                if left > (self.end - self.pos) // size:
                    self.fail("count %d of %r values runs past the end (%d bytes left)" % (left, typ, self.end - self.pos), at)
                p = self.take(left * size, "typed array")
                return np.frombuffer(self.buf, _BIG[typ], left, p).astype(_NATIVE[typ])
            if m == "[" and typ in ("Z", "T", "F"):
                if left > MAX_EMPTY_ELEMENTS:
                    self.fail("count %d of %r values exceeds the limit of %d" % (left, typ, MAX_EMPTY_ELEMENTS), at)
            elif left > self.end - self.pos:   # every entry (an object's: its key) takes at least one byte
                self.fail("count %d runs past the end (%d bytes left)" % (left, self.end - self.pos), at)
        return _Frame(m == "{", left, typ)

    def closes(self, f):
        """Whether the open container f ends here (its count is used up, or its closing marker is next: consumed)."""
        if f.left is not None:
            return f.left == 0
        while True:
            c = self.peek("'%s'" % ("}" if f.obj else "]"))
            if c != "N":
                break
            self.pos += 1
        if c == ("}" if f.obj else "]"):
            self.pos += 1
            return True
        return False

    def value(self):
        """The value starting here, containers read with an explicit stack so that nesting has no depth limit."""
        stack = []
        m = self.marker()
        at = self.pos - 1
        while True:
            if m in "[{":
                v = self.open(m)
                if isinstance(v, _Frame):
                    stack.append(v)
                elif not stack:
                    return v
                else:
                    stack[-1].put(v)
            else:
                v = self.scalar(m, at)
                if not stack:
                    return v
                stack[-1].put(v)
            # the next value of the innermost open container, closing each container that ends here
            while True:
                f = stack[-1]
                if not self.closes(f):
                    break
                stack.pop()
                if not stack:
                    return f.out
                stack[-1].put(f.out)
            if f.obj:
                f.key = self.key()
            if f.typ is not None:
                m, at = f.typ, self.pos
            else:
                m = self.marker()
                at = self.pos - 1


def loads(buf, pos=0):
    """The document encoded in buf[pos:] (bytes-like), which must end where the buffer ends."""
    r = _Reader(buf, pos)
    v = r.value()
    if r.pos != r.end:
        r.fail("%d trailing bytes after the top-level value" % (r.end - r.pos))
    return v


def _count(n):
    return b"L" + struct.pack(">q", n)


def _typed(values, t):
    """`[$t#L n` and the big-endian elements; values the element type cannot hold exactly are refused."""
    if t == "d":
        a = np.asarray(values, np.float64)
        f = a.astype(np.float32)
        if not np.array_equal(f.astype(np.float64), a, equal_nan=True):
            raise XGBoostError("typed 'd' array holds values float32 cannot hold exactly")
    else:
        a = np.asarray(values)
        if a.size and not np.issubdtype(a.dtype, np.integer):
            raise XGBoostError("typed %r array holds non-integer values of %s" % (t, a.dtype))
        f = a.astype(_NATIVE[t])
        if not np.array_equal(f, a):
            raise XGBoostError("typed %r array holds values outside its range" % t)
    return b"".join((b"[$", t.encode(), b"#", _count(f.size), f.astype(_BIG[t]).tobytes()))


def _put(v, out):
    if v is None:
        out.append(b"Z")
    elif isinstance(v, (bool, np.bool_)):
        out.append(b"T" if v else b"F")
    elif isinstance(v, (int, np.integer)):
        if not -2 ** 63 <= int(v) < 2 ** 63:
            raise XGBoostError("integer %d does not fit int64" % int(v))
        out.append(_count(int(v)))
    elif isinstance(v, (float, np.floating)):
        f = np.float32(v)
        exact = float(f) == float(v) or v != v
        out.append(b"d" + struct.pack(">f", f) if exact else b"D" + struct.pack(">d", float(v)))
    elif isinstance(v, str):
        b = v.encode("utf-8")
        out += [b"S", _count(len(b)), b]
    elif isinstance(v, dict):
        out.append(b"{")
        for k, x in v.items():
            if not isinstance(k, str):
                raise XGBoostError("object key %r is not a string" % (k,))
            b = k.encode("utf-8")
            out += [_count(len(b)), b]
            if k in XGBOOST_TYPED and isinstance(x, (list, tuple, np.ndarray)):
                out.append(_typed(x, XGBOOST_TYPED[k]))
            else:
                _put(x, out)
        out.append(b"}")
    elif isinstance(v, (list, tuple, np.ndarray)):
        out.append(b"[")
        for x in v:
            _put(x, out)
        out.append(b"]")
    else:
        raise XGBoostError("cannot encode %s as UBJSON" % type(v).__name__)


def dumps(doc):
    """UBJSON of doc (dicts, lists, str, int, float, bool, None, NumPy arrays and scalars); an array under a key of
    XGBOOST_TYPED is written as a typed array of that element type."""
    out = []
    _put(doc, out)
    return b"".join(out)
