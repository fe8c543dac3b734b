// check.h — what every host-compiled test program shares: CHECK counts every check and prints the first 20 failures;
// test_seed perturbs a program's fixed generator seed by PCLB_TEST_SEED (tools/dev/fuzz_host_tests.sh), unset = the seed.
#pragma once

#include <cstdio>
#include <cstdlib>

static long g_checks = 0, g_fail = 0;
#define CHECK(c, ...) do { ++g_checks; if (!(c)) { if (++g_fail <= 20) { std::printf("FAIL %s:%d %s  ", __FILE__, __LINE__, #c); std::printf(__VA_ARGS__); std::printf("\n"); } } } while (0)

static unsigned test_seed(unsigned fixed)
{
  const char* e = std::getenv("PCLB_TEST_SEED");
  return e && *e ? fixed ^ (2654435761u * static_cast<unsigned>(std::strtoul(e, nullptr, 10))) : fixed;
}
