"""The ctypes mirrors in graphgps_b200/_lib.py against include/gps_b200.h, compiled with the host C compiler: the size
of every mirrored struct and the offset of each of its fields, and the value of every enum constant _lib mirrors.  A
field added, moved or retyped on one side only would otherwise corrupt every call without an error."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from graphgps_b200 import _lib

INCLUDE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "include")

STRUCTS = [_lib.GpsGraph, _lib.GpsBatchNorm, _lib.GpsLinear, _lib.GpsPlanes, _lib.GpsAttnBias, _lib.GpsGat,
           _lib.GpsGenConv, _lib.GpsPna, _lib.GpsBigBird, _lib.GpsLayerArgs, _lib.GpsLayerPlan, _lib.GpsGraphormerArgs,
           _lib.GpsGraphormerPlan, _lib.GpsSanArgs, _lib.GpsSanPlan, _lib.GpsCustomGnnArgs, _lib.GpsCustomGnnPlan,
           _lib.GpsGemmArgs, _lib.GpsRowwiseBn, _lib.GpsRowwiseArgs, _lib.GpsAttnStageArgs]

# header enum prefix -> the _lib name -> value map it must equal (keys upper-cased, "Custom" dropped: CustomGatedGCN is
# GPS_LOCAL_GATEDGCN)
ENUMS = {
    "GPS_LOCAL_": _lib.LOCAL,
    "GPS_GLOBAL_": _lib.GLOBAL,
    "GPS_ACT_": _lib.ACT,
    "GPS_PREC_": _lib.PRECISION,
    "GPS_NORM_": _lib.NORM,
    "GPS_FLAG_": {"GRADS_ZEROED": _lib.FLAG_GRADS_ZEROED, "GRADS_ACCUMULATE": _lib.FLAG_GRADS_ACCUMULATE},
    "GPS_BIGBIRD_": _lib.BIGBIRD_ACT,
    "GPS_CUSTOM_": {"GATEDGCN": _lib.CUSTOM_GATEDGCN, "GINE": _lib.CUSTOM_GINE},
    "GPS_ROWWISE_": _lib.ROWWISE,
    "GPS_ATTN_": _lib.ATTN,
}


@pytest.fixture(scope="module")
def header_layout(tmp_path_factory):
    """{"Struct": size, "Struct.field": offset, "GPS_X_Y": value} as the C compiler lays out the header."""
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no host C compiler")
    hdr = open(os.path.join(INCLUDE, "gps_b200.h")).read()
    consts = sorted(set(re.findall(r"\b(%s)[A-Z0-9_]*\s*=" % "|".join(ENUMS), hdr)))
    names = sorted(set(re.findall(r"\b((?:%s)[A-Z0-9_]+)\s*=" % "|".join(ENUMS), hdr)))
    assert consts == sorted(ENUMS), consts
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "gps_b200.h"', "int main(void) {"]
    for s in STRUCTS:
        t = s.__name__
        lines.append(f'  printf("{t} %zu\\n", sizeof({t}));')
        for f, _ in s._fields_:
            lines.append(f'  printf("{t}.{f} %zu\\n", offsetof({t}, {f}));')
    for n in names:
        lines.append(f'  printf("{n} %d\\n", (int){n});')
    lines += ["  return 0;", "}"]
    d = tmp_path_factory.mktemp("abi_layout")
    src, exe = d / "layout.c", d / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    return {k: int(v) for k, v in (line.split() for line in out.splitlines())}


@pytest.mark.parametrize("struct", STRUCTS, ids=lambda s: s.__name__)
def test_struct_layout_matches_header(header_layout, struct):
    t = struct.__name__
    got = {f: getattr(struct, f).offset for f, _ in struct._fields_}
    want = {f: header_layout[f"{t}.{f}"] for f, _ in struct._fields_}
    assert got == want
    assert C.sizeof(struct) == header_layout[t]


@pytest.mark.parametrize("prefix", sorted(ENUMS))
def test_enum_constants_match_header(header_layout, prefix):
    header = {k[len(prefix):]: v for k, v in header_layout.items() if k.startswith(prefix) and "." not in k}
    mirrored = {k.upper().replace("CUSTOM", ""): v for k, v in ENUMS[prefix].items()}
    assert mirrored == header
