"""CPU oracle of the device-evaluated point lights — TEST INFRASTRUCTURE, like the rest of this package.

libr3_oracle_points.so (r3_oracle_points.c, which includes the shadow-camera oracle r3_oracle_lights.c) links libr3_oracle.so: one handle
through which every r3o_ entry point resolves, the shadow-camera twins and the point-light twins (r3o_set_point_light_sources ...
r3o_readback_point_lights) included."""
import ctypes
import os
import subprocess

from . import _DIR
from . import build as build_oracle
from .anim import CFLAGS

LIB_PATH = os.path.join(_DIR, "libr3_oracle_points.so")


def build(force: bool = False) -> str:
    base = build_oracle()
    src = os.path.join(_DIR, "r3_oracle_points.c")
    srcs = [src, os.path.join(_DIR, "r3_oracle_lights.c"), os.path.join(_DIR, "r3_oracle.h"), base, __file__]
    srcs += [os.path.join(_DIR, "..", "include", f) for f in ("r3_layouts.h", "rend3_b200.h")]
    stale = force or not os.path.exists(LIB_PATH) or any(os.path.exists(s) and os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if stale:
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        cmd = [cc, *CFLAGS, "-shared", "-o", LIB_PATH, src, "-L", _DIR, "-l:libr3_oracle.so", "-Wl,-rpath,$ORIGIN", "-lm", "-lpthread"]
        try:
            subprocess.run(cmd, check=True, capture_output=True, text=True)
        except (subprocess.CalledProcessError, FileNotFoundError) as e:  # keep a prebuilt .so usable on boxes without gcc
            if not os.path.exists(LIB_PATH):
                raise RuntimeError(f"point-light oracle build failed: {getattr(e, 'stderr', e)}")
    return LIB_PATH


def load_points_oracle_backend():
    """A Backend over the oracle with the shadow-camera and point-light entry points.  r3o_set_directional_lights and r3o_set_point_lights
    live in the base oracle, which knows nothing of the sources: this backend marks the directional sources unset before each such call
    and empties the point-light handle table after it, as r3_set_directional_lights and r3_set_point_lights do in the library."""
    from rend3_b200.backend import Backend

    class PointsOracleBackend(Backend):
        def set_directional_lights(self, data: bytes, atlas_w: int, atlas_h: int):
            self.lib.r3o_lights_forget(self.ctx)
            super().set_directional_lights(data, atlas_w, atlas_h)

        def set_point_lights(self, data: bytes):
            super().set_point_lights(data)
            self.lib.r3o_points_forget(self.ctx)

        def close(self):
            if self.ctx:
                self.lib.r3o_points_release(self.ctx)
                self.lib.r3o_lights_release(self.ctx)
            super().close()

    return PointsOracleBackend(ctypes.CDLL(build()), "r3o_", 0)
