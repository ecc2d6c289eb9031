"""Host side of the per-replica hyperparameters: the ctypes mirror of b200sac_hparams."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_hparams_struct_matches_header():
    from distributed_sac_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "b200sac.h")).read()
    body = re.search(r"typedef struct b200sac_hparams \{(.*?)\} b200sac_hparams;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    declared = [n.strip() for decl in body.split(";") if decl.strip() for n in decl.replace("double", "").split(",")]
    assert [name for name, _ in _lib.Hparams._fields_] == declared
    assert all(t is _lib.C.c_double for _, t in _lib.Hparams._fields_)
