"""A quantised matrix's bin layout, dense or CSR, is known by matrix.cu alone.

The split-side launchers (histogram, partition, final assign, DART) take one B2BinRows and pick the kernel for its
layout inside, as the tree walks take one B2RawRows.  The host files get that source from bin_source(m) and never read
the layout's buffers, so a change to a layout touches matrix.cu and the kernel files only.  The host files are host.h
and the .cu files that include it."""
import re

from tests.test_launch_header import HEADER, _declared, _host_files, _source

LAUNCHERS = ["b2_launch_hist", "b2_launch_partition", "b2_launch_final_assign", "b2_launch_dart_margins"]
LAYOUT_NAMES = ["csr_bins", "ebins", "bins_col", "col_stride"]


def test_one_launcher_per_split_side_kernel():
    text = _source(HEADER)
    declared = _declared(text)
    for name in LAUNCHERS:
        assert name in declared, name
        twins = sorted(d for d in declared if d.startswith(name + "_csr"))
        assert not twins, "%s declares layout twins of %s: %s" % (HEADER, name, ", ".join(twins))
        params = re.search(r"\b%s\s*\(([^;{}]*)\)\s*;" % name, text).group(1)
        assert re.match(r"\s*B2BinRows\s+src\b", params), "%s does not take a B2BinRows first: %s" % (name, params)


def test_only_matrix_cu_names_the_bin_layout():
    offenders = []
    for f in _host_files():
        if f == "matrix.cu":
            continue
        names = sorted(set(re.findall(r"\b(%s)\b" % "|".join(LAYOUT_NAMES), _source(f))))
        if names:
            offenders.append("%s (%s)" % (f, ", ".join(names)))
    assert not offenders, "host files other than matrix.cu name the bin layout: " + "; ".join(offenders)
