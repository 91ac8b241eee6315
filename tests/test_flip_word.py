"""The flip word of the placement kernel's steady-state all-reduce (csrc/simon_flip_word.h), checked on the CPU with the kernel's
own helper: every thread encodes (net change of its counted set, its flipped nodes), the words are summed modulo 2^32 as the
cluster's W_SUM reduction sums them, and the sum is decoded.

The flip count must come back exact for every node count a variant accepts (the single-node fast path fires on a total of exactly
1), and the net change exactly where the fast path can read it (one flip, |dc| <= 1) and wherever its field holds it; past that
it may only differ by a multiple of the field's modulus (it then feeds a prediction that the full summary checks).  The 16 / 16
split of the shared-memory variants is also run at the large variant's sizes, where it must fail: Σnf = 65,537 decodes as 1.
"""
import os
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "open-simulator_b200", "csrc")

# The large variant's geometry: 16 CTAs x 320 threads, up to 64 node slots per thread (327,680 nodes); node n of a scenario is
# slot n / 5120 of thread n % 5120.  A check case (N, nf, dc) flips nf of the N nodes, dc of them changing the counted set by
# sign(dc) each; the flips and the counted-set changes are dealt to the threads in node order, so a thread has nf_t <= 64 and
# |dc_t| <= nf_t.  sum_groups() adds the (at most three) distinct thread words times their thread counts; sum_threads() adds
# the words of all threads one by one, at every 4,099th N (257th for the shared-memory split) and at the wrap sizes.
PROGRAM = r"""
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include "simon_flip_word.h"

static const uint32_t T_BIG = 16 * 320, MAX_NPT = 64;

struct Case { uint32_t n, nf; int32_t dc; };

// thread t's share of k items dealt in node order to T threads
static inline uint32_t share(uint32_t k, uint32_t T, uint32_t t) { return k / T + (t < k % T ? 1u : 0u); }

template <class FW> static uint32_t sum_threads(const Case &c, uint32_t T) {
    uint32_t s = 0, m = (uint32_t)(c.dc < 0 ? -c.dc : c.dc);
    for (uint32_t t = 0; t < T; t++) {
        uint32_t nf = share(c.nf, T, t), mt = share(m, T, t);
        if (nf > MAX_NPT || mt > nf) { fprintf(stderr, "bad deal\n"); exit(2); }
        s += FW::enc(c.dc < 0 ? -(int32_t)mt : (int32_t)mt, nf);
    }
    return s;
}

template <class FW> static uint32_t sum_groups(const Case &c, uint32_t T) {
    // thread ranks where the shares change: [0, a) [a, b) [b, T) with a <= b the smaller and larger remainder
    uint32_t m = (uint32_t)(c.dc < 0 ? -c.dc : c.dc), r1 = c.nf % T, r2 = m % T;
    uint32_t cut[4] = {0, r1 < r2 ? r1 : r2, r1 < r2 ? r2 : r1, T};
    uint32_t s = 0;
    for (int g = 0; g < 3; g++) {
        if (cut[g + 1] == cut[g]) continue;
        uint32_t t = cut[g], nf = share(c.nf, T, t), mt = share(m, T, t);
        s += (cut[g + 1] - cut[g]) * FW::enc(c.dc < 0 ? -(int32_t)mt : (int32_t)mt, nf);
    }
    return s;
}

// 0 when the decoded sum is right: nf exact; dc exact when |dc| fits the field (always when nf == 1), else congruent modulo it
template <class FW> static int check_one(const Case &c, uint32_t sum, long *n_exact_dc) {
    const int dc_bits = 32 - FW::NF_BITS;
    const int32_t dc_lim = (1 << (dc_bits - 1)) - 1;
    if (FW::nf(sum) != c.nf) return 1;
    const int32_t got = FW::dc(sum, FW::nf(sum));
    if ((c.dc >= -dc_lim && c.dc <= dc_lim) || c.nf == 1) {
        ++*n_exact_dc;
        return got == c.dc ? 0 : 2;
    }
    return (((uint32_t)got - (uint32_t)c.dc) & ((1u << dc_bits) - 1u)) == 0 ? 0 : 3;
}

// every N in [1, max_n]; Σnf over the listed values <= N (and N itself); Σdc over ±N, the field edges and ±1
template <class FW> static int run(const char *name, uint32_t max_n, uint32_t T, uint32_t thread_stride) {
    const uint32_t nfs[] = {0, 1, 2, 65535, 65536, 65537, 131073};
    long n_cases = 0, n_thread_sums = 0, n_exact_dc = 0, n_bad = 0, n_false_single = 0;
    const int32_t edge = (1 << (31 - FW::NF_BITS)) - 1;
    for (uint32_t n = 1; n <= max_n; n++) {
        const uint32_t tt = n < T ? n : T;
        for (int q = 0; q < 8; q++) {
            const uint32_t nf = q < 7 ? nfs[q] : n;
            if (nf > n || (q < 7 && nf == n)) continue;
            const int32_t dcs[] = {0, 1, -1, 2, -2, edge, -edge, edge + 1, -edge - 1, (int32_t)nf, -(int32_t)nf, (int32_t)nf - 1,
                                   1 - (int32_t)nf};
            for (int32_t dc : dcs) {
                if ((uint32_t)(dc < 0 ? -dc : dc) > nf) continue;
                const Case c{n, nf, dc};
                uint32_t s = sum_groups<FW>(c, tt);
                if (n % thread_stride == 0 || n == max_n || n == 65536 || n == 65537 || n == 131073) {
                    if (sum_threads<FW>(c, tt) != s) { fprintf(stderr, "%s: thread sums disagree\n", name); return 2; }
                    n_thread_sums++;
                }
                int e = check_one<FW>(c, s, &n_exact_dc);
                n_cases++;
                n_false_single += FW::nf(s) == 1 && nf != 1;    // would take the single-node flip fast path
                if (e && n_bad++ < 5)
                    printf("%s FAIL kind=%d N=%u nf=%u dc=%d -> nf=%u dc=%d\n", name, e, n, nf, dc, FW::nf(s), FW::dc(s, FW::nf(s)));
            }
        }
    }
    printf("%s cases=%ld thread_sums=%ld exact_dc=%ld false_single=%ld bad=%ld\n", name, n_cases, n_thread_sums, n_exact_dc,
           n_false_single, n_bad);
    return n_bad ? 1 : 0;
}

int main(int argc, char **argv) {
    const int which = argc > 1 ? atoi(argv[1]) : 0;
    if (which == 0) return run<SkFlipWord<true>>("large", 327680, T_BIG, 4099);
    if (which == 1) return run<SkFlipWord<false>>("shared", 20480, T_BIG, 257);
    return run<SkFlipWord<false>>("split16_at_large_sizes", 327680, T_BIG, 4099);   // must fail
}
"""


@pytest.fixture(scope="module")
def prog(tmp_path_factory):
    cxx = shutil.which("g++") or shutil.which("c++")
    assert cxx, "a C++ compiler is needed to build the flip-word check"
    d = tmp_path_factory.mktemp("flip_word")
    src, exe = d / "flip_word.cpp", d / "flip_word"
    src.write_text(PROGRAM)
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I", CSRC, str(src), "-o", str(exe)])
    return str(exe)


def _run(prog, which):
    r = subprocess.run([prog, str(which)], capture_output=True, text=True, timeout=600)
    assert r.returncode in (0, 1), r.stderr
    fields = dict(kv.split("=") for kv in r.stdout.strip().splitlines()[-1].split()[1:])
    return r.returncode, {k: int(v) for k, v in fields.items()}, r.stdout


def test_large_variant_flip_word_is_exact_up_to_327680_nodes(prog):
    rc, f, out = _run(prog, 0)
    assert rc == 0 and f["bad"] == 0 and f["false_single"] == 0, out
    assert f["cases"] > 327680 * 8 and f["thread_sums"] > 80 * 8 and f["exact_dc"] > 327680 * 8, out


def test_shared_memory_variants_flip_word_is_exact_up_to_20480_nodes(prog):
    rc, f, out = _run(prog, 1)
    assert rc == 0 and f["bad"] == 0, out
    assert f["cases"] > 20480 * 8 and f["exact_dc"] == f["cases"], out     # 16 bits hold every |dc| <= 20,480


def test_16_bit_flip_count_wraps_at_the_large_variant_sizes(prog):
    """The check has teeth: the shared-memory variants' 16 / 16 split, run at the large variant's sizes, decodes 65,537 flips
    as 1 (and 65,536 as 0)."""
    rc, f, out = _run(prog, 2)
    assert rc == 1 and f["bad"] > 0, out
    assert "N=65536 nf=65536 dc=0 -> nf=0 " in out, out
    assert f["false_single"] > 0, out      # Σnf = 65,537, 131,073, ... taken for a single flip
