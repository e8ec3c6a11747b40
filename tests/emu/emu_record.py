"""TEST INFRASTRUCTURE ONLY. The tester-record entry points (mapdn_record_layout / mapdn_record / mapdn_step_record) of
the emulated library (tests/emu/emu_env.py), as an EmuEnv with three more methods."""
import ctypes as C

import numpy as np

from emu_env import EmuEnv, _ptr, lib


def record_lib():
    L = lib()
    vp = C.c_void_p
    L.mapdn_record_layout.argtypes = [vp, vp, vp]
    L.mapdn_record.argtypes = [vp, vp, C.c_int64, vp]
    L.mapdn_step_record.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, vp, C.c_int64, vp]
    return L


class EmuRecordEnv(EmuEnv):
    def record_layout(self):
        off, row = (C.c_int32 * 6)(), C.c_int32(0)
        self._chk(record_lib().mapdn_record_layout(self._h, off, C.byref(row)))
        return [int(o) for o in off], int(row.value)

    def record(self, out):
        """mapdn_record into ``out`` (a [B, >= row_len] fp64 array, any row stride)."""
        self._chk(record_lib().mapdn_record(self._h, _ptr(out), out.strides[0] // 8, None))
        return out

    def step_record(self, actions, out, add_noise=True):
        """mapdn_step_record: the step of :meth:`step`, plus the record row of every env in ``out``."""
        a = np.ascontiguousarray(actions, np.float64)
        self._chk(record_lib().mapdn_step_record(self._h, _ptr(a), int(add_noise), _ptr(self.reward), _ptr(self.term),
                                                 _ptr(self.info), _ptr(self.obs), _ptr(out), out.strides[0] // 8, None))
        return self.reward, self.term, self.info
