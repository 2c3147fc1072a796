"""The packed results of dfvo_essential_tail (with the dfvo_scale_ransac io block as its prefix) and dfvo_pnp_tail have one
definition, the DFVO_TAIL_* / DFVO_PNP_* enums of include/dfvo_b200.h; b200/native.py mirrors it (runs without a GPU)."""
import os
import re

from b200 import native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_offsets():
    txt = open(os.path.join(ROOT, "include", "dfvo_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    out = {}
    for body in re.findall(r"\benum\s*\{(.*?)\}", txt, flags=re.S):
        for name, value in re.findall(r"\b(DFVO_(?:TAIL|PNP)_[A-Z0-9_]+)\s*=\s*(\d+)", body):
            out[name] = int(value)
    return out


def test_native_mirrors_header_offsets():
    hdr = header_offsets()
    assert len(hdr) >= 20
    mirrored = {k: getattr(native, k) for k in dir(native) if re.fullmatch(r"DFVO_(TAIL|PNP)_[A-Z0-9_]+", k)}
    assert mirrored == hdr


def test_layout_fields_are_contiguous():
    h = header_offsets()
    assert [h["DFVO_TAIL_SCALE"], h["DFVO_TAIL_STATUS"], h["DFVO_TAIL_TRIALS"], h["DFVO_TAIL_INLIERS"], h["DFVO_TAIL_MT"]] == [0, 1, 2, 3, 4]
    assert 2 * h["DFVO_TAIL_MT_DOUBLES"] >= 625                       # key[624], pos as uint32
    assert h["DFVO_TAIL_SCALE_IO"] == h["DFVO_TAIL_MT"] + h["DFVO_TAIL_MT_DOUBLES"] == h["DFVO_TAIL_BEST"]
    singles = ["DFVO_TAIL_BEST", "DFVO_TAIL_VALID", "DFVO_TAIL_HGRIC", "DFVO_TAIL_CHEIR", "DFVO_TAIL_NVALID", "DFVO_TAIL_GATE",
               "DFVO_TAIL_RT"]
    assert [h[k] for k in singles] == list(range(h["DFVO_TAIL_BEST"], h["DFVO_TAIL_BEST"] + len(singles)))
    assert h["DFVO_TAIL_EGRIC"] == h["DFVO_TAIL_RT"] + 12
    assert [h["DFVO_PNP_BEST"], h["DFVO_PNP_INLIERS"], h["DFVO_PNP_RVEC"]] == [0, 1, 2]
    assert h["DFVO_PNP_TVEC"] == h["DFVO_PNP_RVEC"] + 3 and h["DFVO_PNP_INFO"] == h["DFVO_PNP_TVEC"] + 3


def test_result_sizes_come_from_the_header():
    h = header_offsets()
    for R in (1, 5, 32):
        assert native.tail_result_doubles(R) == h["DFVO_TAIL_EGRIC"] + 5 * R
        assert native.pnp_result_doubles(R) == h["DFVO_PNP_INFO"] + 4 * R
    assert native.DFVO_TAIL_SCALE_IO == h["DFVO_TAIL_SCALE_IO"]
