#!/usr/bin/env python3
"""ThreadSanitizer pass over the multi-stream instantiations of the match kernels (tests/emu, test infrastructure).

    python tests/emu/run_tsan_multi.py

Builds tests/emu/emu_multi_driver.cpp like run_tsan.py builds emu_driver.cpp (-fsanitize=thread, -DSB_EMU_THREADS: one
OS thread per CUDA thread) and runs the checks of tests/test_kernel_emulation_multi.py under it: every kernel with
both screening loops, with and without the debug curve, the persistent pair kernel walking across streams, the
multi-stream forward kernel.  Exit code 0 and "0 races" expected."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, 'tests', 'emu', '_build', 'libsb_emu_multi_tsan.so')
LOG = os.path.join(ROOT, 'tests', 'emu', '_build', 'tsan_multi.log')


def main():
    if os.environ.get('SB_EMU_TSAN_CHILD') != '1':
        from tests.test_kernel_emulation_multi import build_lib
        build_lib(LIB, ['-g', '-fsanitize=thread', '-DSB_EMU_THREADS'], load=False)
        tsan = subprocess.check_output(['gcc', '-print-file-name=libtsan.so']).decode().strip()
        env = dict(os.environ, SB_EMU_TSAN_CHILD='1', LD_PRELOAD=tsan, TSAN_OPTIONS='halt_on_error=0 history_size=2 log_path=' + LOG)
        for f in os.listdir(os.path.dirname(LOG)):
            if f.startswith('tsan_multi.log'):
                os.remove(os.path.join(os.path.dirname(LOG), f))
        rc = subprocess.call([sys.executable, os.path.abspath(__file__)], env=env)
        races = 0
        for f in os.listdir(os.path.dirname(LOG)):
            if f.startswith('tsan_multi.log'):
                races += open(os.path.join(os.path.dirname(LOG), f)).read().count('WARNING: ThreadSanitizer')
        print('%d races reported (logs: %s.*), child exit code %d' % (races, LOG, rc))
        return 1 if races or rc else 0

    import ctypes
    from tests.test_kernel_emulation_multi import check_multi
    check_multi(ctypes.CDLL(LIB), log=lambda *a: print(*a, flush=True))
    return 0


if __name__ == '__main__':
    sys.exit(main())
