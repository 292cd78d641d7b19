"""glibc's random() in lsdgpu_rand_state (CPU): lsdgpu_rand_state_seed + lsdgpu_rand_state_advance against the process's own libc
random() in all five state types, the jump-ahead against single steps, the layout of glibc's state buffers that the C++ adapter
reads, and the rejection of bad states.  These host hooks share their generator (csrc/rand.cuh) with the device draws of
lsdgpu_depth_init_random."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from lsd_slam_b200 import abi

# initstate() buffer size -> state type (stdlib/random.c: < 32 TYPE_0, < 64 TYPE_1, < 128 TYPE_2, < 256 TYPE_3, else TYPE_4)
SIZES = {0: 8, 1: 32, 2: 64, 3: 128, 4: 256}
DEG = {0: 1, 1: 7, 2: 15, 3: 31, 4: 63}
SEEDS = [0, 1, 12345, 2**31 - 1, 2**32 - 1]

# draws from the process's libc random() in a given state type; the previous state is put back afterwards, so the rest of the
# test process (srand / rand of the other tests) is unaffected
HELPER = r"""
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
static int32_t buf[64];
int draws(unsigned seed, int size, long n, int32_t* out)
{
    char* old = initstate(seed, (char*)buf, size);
    if (!old) return -1;
    for (long i = 0; i < n; i++) out[i] = (int32_t)random();
    setstate(old);
    return 0;
}
/* the live state after k draws, read the way the adapter reads it: initstate() returns the word before the live table */
int snapshot(unsigned seed, int size, long k, int32_t* words)
{
    int32_t tmp[32];
    char* old = initstate(seed, (char*)buf, size);
    if (!old) return -1;
    for (long i = 0; i < k; i++) (void)random();
    int32_t* live = (int32_t*)initstate(1, (char*)tmp, sizeof tmp);
    memcpy(words, live, 64 * 4);
    setstate((char*)live);
    setstate(old);
    return 0;
}
"""


@pytest.fixture(scope="module")
def libc_random(tmp_path_factory):
    d = tmp_path_factory.mktemp("libc_random")
    (d / "h.c").write_text(HELPER)
    so = d / "libh.so"
    r = subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-o", str(so), str(d / "h.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(str(so))
    L.draws.argtypes = [C.c_uint, C.c_int, C.c_long, C.POINTER(C.c_int32)]
    L.snapshot.argtypes = [C.c_uint, C.c_int, C.c_long, C.POINTER(C.c_int32)]
    return L


def _libc(L, seed, t, n):
    out = np.zeros(n, np.int32)
    assert L.draws(seed, SIZES[t], n, out.ctypes.data_as(C.POINTER(C.c_int32))) == 0
    return out


@pytest.mark.parametrize("t", range(5))
def test_seed_and_advance_equal_libc_random(libc_random, t):
    n = 2_000_000
    for seed in SEEDS:
        want = _libc(libc_random, seed, t, n)
        st = abi.RandState.from_seed(seed, t)
        got = st.advance(n)
        assert np.array_equal(got, want), (t, seed, int(np.argmax(got != want)))


@pytest.mark.parametrize("t", range(5))
def test_jump_then_steps_equals_steps(t):
    m = 1000
    for n in sorted({0, 1, max(DEG[t] - 1, 0), DEG[t], 10**6 + 7}):
        a = abi.RandState.from_seed(777, t)
        b = a.copy()
        assert a.advance(n, values=False) is None
        tail = a.advance(m)
        ref = b.advance(n + m)
        assert np.array_equal(tail, ref[n:]), (t, n)
        assert a == b, (t, n)                     # same table and rear index


@pytest.mark.parametrize("t", range(5))
def test_state_layout_of_glibc_buffers(libc_random, t):
    """initstate() returns the word before the live table: 5 * rear + type (TYPE_0: 0), then the table -- lsdgpu_rand_state's
    (type, rear, r) is that word decoded"""
    for k in (0, 1, 3 * DEG[t] + 2, 12345):
        w = np.zeros(64, np.int32)
        assert libc_random.snapshot(4321, SIZES[t], k, w.ctypes.data_as(C.POINTER(C.c_int32))) == 0
        st = abi.RandState.from_seed(4321, t)
        st.advance(k, values=False)
        assert int(w[0]) % 5 == t and int(w[0]) // 5 == st.rear, (t, k, int(w[0]), st.rear)
        assert np.array_equal(w[1:1 + DEG[t]].view(np.uint32), np.array(st.r[:DEG[t]], np.uint32)), (t, k)


def test_bad_states_are_rejected():
    L = abi.load()
    st = abi.RandState()
    assert L.lsdgpu_rand_state_seed(5, 1, C.byref(st)) != 0
    assert L.lsdgpu_rand_state_seed(-1, 1, C.byref(st)) != 0
    assert L.lsdgpu_rand_state_seed(3, 1, None) != 0
    for t, rear in ((-1, 0), (5, 0), (0, 1), (1, 7), (2, 15), (3, 31), (4, 63), (3, -1)):
        st = abi.RandState.from_seed(9, min(max(t, 0), 4))
        st.type, st.rear = t, rear
        before = bytes(st)
        with pytest.raises(ValueError):
            st.advance(10)
        with pytest.raises(ValueError):
            st.advance(10, values=False)
        assert bytes(st) == before
    st = abi.RandState.from_seed(9)
    with pytest.raises(ValueError):
        st.advance(-1, values=False)
