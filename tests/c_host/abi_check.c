/* The C-ABI header must be consumable by a plain C99 compiler (no C++, no CUDA headers): this file is compiled with
 * `gcc -std=c99 -pedantic -Werror -c` by tests/test_host_cpu.py.  It also pins the descriptor layouts the ctypes binding
 * mirrors (omg_b200/_lib.py) through sizeof prints the test compares. */
#include <stdio.h>

#include "omg_b200.h"

int main(void) {
    omg_gemm_desc g;
    omg_attn_desc a;
    omg_fuse_desc f;
    omg_solver_desc s;
    omg_plan* p = 0;
    (void)g;
    (void)a;
    (void)f;
    (void)s;
    (void)p;
    printf("%u %u %u %u %u %u\n", (unsigned)sizeof(omg_view4), (unsigned)sizeof(omg_seg),
           (unsigned)sizeof(omg_gemm_desc), (unsigned)sizeof(omg_attn_desc), (unsigned)sizeof(omg_fuse_desc),
           (unsigned)sizeof(omg_solver_desc));
    return 0;
}
