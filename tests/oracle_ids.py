"""The oracle's ID frames (oracle/forma_oracle_ids.cpp, libforma_oracle_ids.so): bound into the
oracle's Api as `renderer_render_ids`, so that `Renderer.render_ids` of the oracle binding
renders the ID frame of an oracle composition."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE, "libforma_oracle_ids.so")


def attach(oracle_api):
    if not hasattr(oracle_api, "renderer_render_ids"):
        if not os.path.exists(LIB):
            subprocess.check_call(["make", "-C", ORACLE, "-f", "ids.mk"])
        oracle_api.attach(C.CDLL(LIB), ("renderer_render_ids",))
    return oracle_api
