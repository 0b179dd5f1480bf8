"""ctypes wrapper of tests/channel_oracle.c, the CPU restatement of the random-walk StoreChannelData line — TEST
INFRASTRUCTURE ONLY.  The C file is compiled on first use into a temporary directory (the tree may be read-only) and
linked against the CPU oracle's library for its encoding/json string rule (orc_json_string)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

from distributed_crawler_b200 import abi
from oracle import pyoracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        oracle_so = pyoracle.build()
        src = os.path.join(_HERE, "channel_oracle.c")
        with open(src, "rb") as f:
            tag = hashlib.sha256(f.read() + oracle_so.encode()).hexdigest()[:16]
        out_dir = os.path.join(tempfile.gettempdir(), f"tgi_channel_oracle_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        so = os.path.join(out_dir, f"libchannel_oracle_{tag}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            oracle_dir = os.path.dirname(oracle_so)
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared",
                                   "-I", os.path.join(_ROOT, "include"), "-I", oracle_dir, "-o", tmp, src,
                                   "-L", oracle_dir, "-ltgoracle", f"-Wl,-rpath,{oracle_dir}"])
            os.replace(tmp, so)
        C.CDLL(oracle_so, mode=C.RTLD_GLOBAL)
        L = C.CDLL(so)
        L.chorc_create.restype = C.c_void_p
        L.chorc_destroy.argtypes = [C.c_void_p]
        L.chorc_destroy.restype = None
        L.chorc_channel_batch.argtypes = [C.c_void_p, C.POINTER(abi.ChBatchC), C.c_uint32, C.POINTER(pyoracle.OrcResultC)]
        _LIB = L
    return _LIB


class ChannelOracle:
    """the StoreChannelData lines of a pack.pack_channels batch, as pyoracle.Result"""

    def __init__(self):
        self.h = lib().chorc_create()

    def close(self):
        if getattr(self, "h", None):
            lib().chorc_destroy(self.h)
            self.h = None

    __del__ = close

    def channel(self, batch, run_flags=abi.RUN_JSONL) -> pyoracle.Result:
        d = batch.descriptor()
        r = pyoracle.OrcResultC()
        rc = lib().chorc_channel_batch(self.h, C.byref(d), run_flags, C.byref(r))
        if rc != 0:
            raise pyoracle.OracleError(rc, "chorc_channel_batch")
        return pyoracle.result_from_c(r)
