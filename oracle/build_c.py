"""gcc build of the oracle's C restatement (oracle/c/oracle_kernels.c) -> oracle/_c/liboracle.so.  TEST INFRASTRUCTURE."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'c', 'oracle_kernels.c')
OUT = os.path.join(HERE, '_c', 'liboracle.so')


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if force or not os.path.exists(OUT) or os.path.getmtime(OUT) < os.path.getmtime(SRC):
        subprocess.check_call(['gcc', '-O2', '-ffp-contract=off', '-fPIC', '-shared', '-fopenmp', '-o', OUT, SRC, '-lm'])
    return OUT


def load():
    import ctypes
    return ctypes.CDLL(build())


if __name__ == '__main__':
    print(build(force=True))
