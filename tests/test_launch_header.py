"""The kernel launchers are declared once, in csrc/launch.h, and both sides compile against it.

The launchers have C linkage, so a prototype kept apart from its definition links even when the two disagree, and the
kernel then reads shifted arguments at run time.  With one header included by every host file that calls a launcher and
by every defining file, a mismatch is a compile error.  These checks keep it that way: every b2_* function a kernel file
defines for the host is declared in the header and nowhere else.  The host files are host.h and the .cu files that
include it (engine.cu, tree.cu, ...)."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "xgboost_ray_b200", "csrc")
HEADER = "launch.h"


def _source(name):
    text = open(os.path.join(CSRC, name)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return re.sub(r"//[^\n]*", "", text)


def _extern_c_blocks(text):
    for m in re.finditer(r'extern\s+"C"\s*\{', text):
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(text[i], 0)
            i += 1
        yield text[m.end():i - 1]


def _top_level(block):
    """the text of an extern "C" block outside every function body"""
    out, depth = [], 0
    for c in block:
        if c == "}":
            depth -= 1
        if depth == 0:
            out.append(c)
        if c == "{":
            depth += 1
    return "".join(out)


def _defined(text):
    names = set()
    for block in _extern_c_blocks(text):
        names.update(re.findall(r"\b(b2_\w+)\s*\([^;{}]*\)\s*\{", _top_level(block)))
    return names


def _declared(text):
    names = set()
    for block in _extern_c_blocks(text):
        names.update(re.findall(r"\b(b2_\w+)\s*\([^;{}]*\)\s*;", _top_level(block)))
    return names


def _kernel_files():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _includes(text, name):
    return re.search(r'^\s*#\s*include\s+"%s"' % re.escape(name), text, re.M) is not None


def _host_files():
    files = ["host.h"] + [f for f in _kernel_files() if _includes(_source(f), "host.h")]
    assert "engine.cu" in files and len(files) >= 8, files
    return files


def _calls_launcher(text, launchers):
    return any(name in launchers for name in re.findall(r"\b(b2_\w+)\s*\(", text))


def test_header_declares_exactly_the_defined_launchers():
    defined = {}
    for f in _kernel_files():
        for name in _defined(_source(f)):
            assert name not in defined, "%s is defined in both %s and %s" % (name, defined[name], f)
            defined[name] = f
    declared = _declared(_source(HEADER))
    assert len(defined) >= 80
    missing = sorted(set(defined) - declared)
    assert not missing, "defined in an extern \"C\" block but not declared in %s: %s" % (
        HEADER, ", ".join("%s (%s)" % (n, defined[n]) for n in missing))
    stale = sorted(declared - set(defined))
    assert not stale, "declared in %s but defined by no kernel file: %s" % (HEADER, ", ".join(stale))


def test_defining_files_and_engine_include_the_header():
    launchers = _declared(_source(HEADER))
    users = [f for f in _kernel_files() if _defined(_source(f))]
    users += [f for f in _host_files() if _calls_launcher(_source(f), launchers)]
    assert "engine.cu" in users and "tree.cu" in users
    for f in users:
        assert _includes(_source(f), HEADER), "%s does not include %s" % (f, HEADER)


def test_engine_keeps_no_launcher_prototypes():
    abi = []
    for f in _host_files():
        text = _source(f)
        local = sorted(_declared(text) | _defined(text) | set(re.findall(r'extern\s+"C"\s+[^{;]*?\b(b2_\w+)\s*\(', text)))
        assert not local, "%s declares launchers of its own: %s" % (f, ", ".join(local))
        abi += [(f, block) for block in _extern_c_blocks(text)]
    # the only extern "C" block of the host files is the C ABI of include/b2hist.h, in engine.cu
    assert len(abi) == 1 and abi[0][0] == "engine.cu", [f for f, _ in abi]
    assert re.search(r"\bint\s+B2_BoosterCreate\s*\(", abi[0][1])
