#!/usr/bin/env python3
"""ThreadSanitizer pass over the persistent walk of k_forward_quad (tests/emu/emu_forward_driver.cpp, test
infrastructure), like tests/emu/run_tsan.py does for the match kernels.

    python tests/emu/run_tsan_forward.py

Builds the driver with -fsanitize=thread -DSB_EMU_THREADS (one OS thread per CUDA thread, std::barrier for bar.sync)
and runs the cases of tests/test_kernel_emulation_persistent.py: one CTA per row against 1, 2 and 3 CTAs walking
block rows past the end of a stream, template partitions across query boundaries (the CTA-wide query search
re-uses one shared-memory word per step) and the rows of several streams.  A shared-memory access the kernel's
barriers do not order -- the FFT buffer re-used by the next row, the search word -- shows up as a data race.  Exit
code 0 and "0 races" expected.  Re-executes itself under LD_PRELOAD=libtsan.so (the interpreter is not instrumented)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
LIB = os.path.join(ROOT, 'tests', 'emu', '_build', 'libsb_emu_forward_tsan.so')
LOG = os.path.join(ROOT, 'tests', 'emu', '_build', 'tsan_forward.log')


def main():
    if os.environ.get('SB_EMU_TSAN_CHILD') != '1':
        import tests.test_kernel_emulation_persistent as P
        P.build(LIB, ['-g', '-fsanitize=thread', '-DSB_EMU_THREADS'])
        tsan = subprocess.check_output(['gcc', '-print-file-name=libtsan.so']).decode().strip()
        env = dict(os.environ, SB_EMU_TSAN_CHILD='1', LD_PRELOAD=tsan, TSAN_OPTIONS='halt_on_error=0 history_size=2 log_path=' + LOG)
        for f in os.listdir(os.path.dirname(LOG)):
            if f.startswith('tsan_forward.log'):
                os.remove(os.path.join(os.path.dirname(LOG), f))
        rc = subprocess.call([sys.executable, os.path.abspath(__file__)], env=env)
        races = 0
        for f in os.listdir(os.path.dirname(LOG)):
            if f.startswith('tsan_forward.log'):
                races += open(os.path.join(os.path.dirname(LOG), f)).read().count('WARNING: ThreadSanitizer')
        print('%d races reported (logs: %s.*), child exit code %d' % (races, LOG, rc))
        return 1 if races or rc else 0

    import numpy as np
    import tests.test_kernel_emulation_persistent as P
    walk = P.load(LIB)
    P.test_block_rows_do_not_depend_on_the_grid(walk, np.uint8)
    print('block rows ok', flush=True)
    P.test_partition_rows_do_not_depend_on_the_grid(walk)
    print('template partitions ok', flush=True)
    P.test_multi_stream_rows_do_not_depend_on_the_grid(walk)
    print('multi-stream rows ok', flush=True)
    return 0


if __name__ == '__main__':
    sys.exit(main())
