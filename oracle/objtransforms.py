"""CPU oracle of the bulk object-transform entry points — TEST INFRASTRUCTURE, like the rest of this package.

libr3_oracle_objtransforms.so (r3_oracle_objtransforms.c, which includes the object-animation oracle and through it the skeletal one)
links libr3_oracle.so: one handle through which every r3o_ entry point resolves, r3o_set_object_mesh_spheres and
r3o_set_object_transforms included."""
import ctypes
import os
import subprocess

from . import _DIR
from . import build as build_oracle
from .anim import CFLAGS

LIB_PATH = os.path.join(_DIR, "libr3_oracle_objtransforms.so")


def build(force: bool = False) -> str:
    base = build_oracle()
    src = os.path.join(_DIR, "r3_oracle_objtransforms.c")
    srcs = [src, os.path.join(_DIR, "r3_oracle_objanim.c"), os.path.join(_DIR, "r3_oracle_anim.c"), os.path.join(_DIR, "r3_oracle.h"), base, __file__]
    srcs += [os.path.join(_DIR, "..", "include", f) for f in ("r3_layouts.h", "rend3_b200.h", "r3_anim_check.h")]
    stale = force or not os.path.exists(LIB_PATH) or any(os.path.exists(s) and os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if stale:
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        cmd = [cc, *CFLAGS, "-shared", "-o", LIB_PATH, src, "-L", _DIR, "-l:libr3_oracle.so", "-Wl,-rpath,$ORIGIN", "-lm", "-lpthread"]
        try:
            subprocess.run(cmd, check=True, capture_output=True, text=True)
        except (subprocess.CalledProcessError, FileNotFoundError) as e:  # keep a prebuilt .so usable on boxes without gcc
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(f"object transform oracle build failed: {getattr(e, 'stderr', e)}")
    return LIB_PATH


def load_objtransforms_oracle_backend():
    """A Backend over the oracle with the animation and bulk-transform entry points; closing it drops the three side states."""
    from rend3_b200.backend import Backend

    class ObjTransformsOracleBackend(Backend):
        def close(self):
            if self.ctx:
                self.lib.r3o_objtransforms_release(self.ctx)
                self.lib.r3o_objanim_release(self.ctx)
                self.lib.r3o_anim_release(self.ctx)
            super().close()

    return ObjTransformsOracleBackend(ctypes.CDLL(build()), "r3o_", 0)
