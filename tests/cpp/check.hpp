// check.hpp -- the failure count of a C++ host-layer test program.  CHECK(cond) prints each failed condition with its
// file and line and counts it; main ends with `return report();`, which prints the verdict that
// tests/test_gpu_cpp_host.py looks for and gives the exit code.
#pragma once
#include <cstdio>

static int failures = 0;
#define CHECK(cond)                                                                 \
    do {                                                                            \
        if (!(cond)) { std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #cond); failures++; } \
    } while (0)

static int report() {
    if (failures) { std::printf("%d checks failed\n", failures); return 1; }
    std::printf("all checks passed\n");
    return 0;
}
