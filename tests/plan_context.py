"""A dry-run planning context (b200_plan_begin) for the CPU tests and the golden generators.

The library plans every call made on it -- checks, kernel choice, tensor maps, launch geometry -- and records the plan as text
instead of touching a device.  Each test file's Planner subclasses PlanContext with the calls it makes.
"""
import ctypes as C

from cubecl_b200 import _ffi


class PlanContext:
    def __init__(self, sms=132, options=None):   # 132 SMs: H100 SXM
        self.lib = _ffi.load()
        self.ctx = C.c_void_p()
        _ffi.check(self.lib.b200_plan_begin(int(sms), C.byref(self.ctx)))
        try:
            for key, value in (options or {}).items():
                self.option(key, value)
        except Exception:
            self.close()
            raise

    def text(self) -> str:
        """Everything planned in this context so far."""
        need = C.c_size_t()
        _ffi.check(self.lib.b200_plan_text(self.ctx, None, 0, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        _ffi.check(self.lib.b200_plan_text(self.ctx, buf, need.value, None))
        return buf.value.decode()

    def option(self, key, value):
        _ffi.check(self.lib.b200_set_option(self.ctx, key.encode(), str(value).encode()))

    def close(self):
        self.lib.b200_destroy(self.ctx)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
