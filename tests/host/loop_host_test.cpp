// loop_host_test.cpp — the ICP loop's decisions as k_solve's tail makes them (pcl_b200/csrc/solve_body.inc): the
// convergence criteria (icp_kernels.cuh: has_converged_dev) and the composition final = T_k * final (mat4_mul_dev),
// compiled for the HOST and replayed on sequences that tests/test_loop_reference.py writes.  The program only records;
// the Python test compares every record with its plain restatement of PCL's source.  CPU only.
//
// usage: loop_host_test <in> <out>   (without arguments: seeded random sequences, replayed and checked for the loop's
//        invariants only, for the sanitizer, thread-schedule and fuzz scripts of tools/dev)
//   in : int32 n_cases, then per case
//          int32 scalar_is_double, max_iterations, failure_after_max_iter, max_iterations_similar, n_steps
//          double rot_eps, trans_eps, rel_mse, abs_mse, prev_mse (the criteria's value when the align starts)
//          double final[16] (the guess, row-major, already in Scalar)
//          per step: int32 ok (at least 3 pairs), double mse, double T[16] (T_k in Scalar)
//   out: per case int32 n_recorded, then per recorded step
//          int32 state, converged, iterations, iterations_similar; double prev_mse; double final[16]
// A case stops recording at the first step that leaves the state other than NOT_CONVERGED, as the loop stops there.
#define PCLB_HOST_EXTRA_SHIMS "warp_emu.h"
#define PCLB_HOST_EMULATION 1
#include "host_index.h"
#include "check.h"

#include <cfloat>
#include <fstream>
#include <random>
#include <sstream>

static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

#include "../../pcl_b200/csrc/icp_kernels.cuh"

template <typename T> static T rd(std::istream& in)
{
  T v;
  in.read(reinterpret_cast<char*>(&v), sizeof(T));
  return v;
}
template <typename T> static void wr(std::ostream& out, const T& v) { out.write(reinterpret_cast<const char*>(&v), sizeof(T)); }

static long long replay(std::istream& in, std::ostream& out)
{
  const int n_cases = rd<int32_t>(in);
  long long steps = 0;
  for (int c = 0; c < n_cases && in; ++c) {
    CritParams P{};
    P.scalar_is_double = rd<int32_t>(in);
    P.max_iterations = rd<int32_t>(in);
    P.failure_after_max_iter = rd<int32_t>(in);
    P.max_iterations_similar = rd<int32_t>(in);
    const int n_steps = rd<int32_t>(in);
    P.rot_eps = rd<double>(in);
    P.trans_eps = rd<double>(in);
    P.rel_mse = rd<double>(in);
    P.abs_mse = rd<double>(in);
    // the loop state as icp_set_source leaves it (icp.cu: icp_reset_state)
    LoopCtrl L;
    std::memset(&L, 0, sizeof(L));
    L.state = PCLB200_CONV_NOT_CONVERGED;
    L.prev_mse = rd<double>(in);
    for (int i = 0; i < 16; ++i)
      L.final_T[i] = rd<double>(in);
    std::vector<char> rec;
    int recorded = 0;
    for (int k = 0; k < n_steps; ++k) {
      const int ok = rd<int32_t>(in);
      const double mse = rd<double>(in);
      double T[16];
      for (int i = 0; i < 16; ++i)
        T[i] = rd<double>(in);
      if (L.done)
        continue;
      // solve_body.inc's tail, the part that decides
      L.mse = mse;
      if (!ok) {
        L.state = PCLB200_CONV_NO_CORRESPONDENCES;
        L.converged = 0;
        L.done = 1;
      }
      else {
        for (int i = 0; i < 16; ++i)
          L.last_T[i] = T[i];
        if (P.scalar_is_double)
          mat4_mul_dev<double>(L.last_T, L.final_T, L.final_T);
        else
          mat4_mul_dev<float>(L.last_T, L.final_T, L.final_T);
        ++L.iterations;
        L.converged = (P.scalar_is_double ? has_converged_dev<double>(L, P, L.last_T) : has_converged_dev<float>(L, P, L.last_T)) ? 1 : 0;
        if (L.state != PCLB200_CONV_NOT_CONVERGED)
          L.done = 1;
      }
      const int32_t head[4] = {L.state, L.converged, L.iterations, L.iterations_similar};
      const char* h = reinterpret_cast<const char*>(head);
      rec.insert(rec.end(), h, h + sizeof(head));
      const char* pm = reinterpret_cast<const char*>(&L.prev_mse);
      rec.insert(rec.end(), pm, pm + 8);
      const char* f = reinterpret_cast<const char*>(L.final_T);
      rec.insert(rec.end(), f, f + sizeof(L.final_T));
      ++recorded;
      ++steps;
    }
    wr(out, (int32_t)recorded);
    out.write(rec.data(), (std::streamsize)rec.size());
  }
  CHECK(in.good(), "truncated input");
  std::printf("%d cases, %lld steps recorded\n", n_cases, steps);
  return steps;
}

// random criteria and steps around the thresholds; every recorded case must be a loop's history
static void self_test()
{
  std::mt19937_64 g(test_seed(20261019u));
  std::uniform_real_distribution<double> u(0.0, 1.0);
  std::stringstream in, out;
  const int n_cases = 2000;
  wr(in, (int32_t)n_cases);
  for (int c = 0; c < n_cases; ++c) {
    const int n_steps = 1 + (int)(g() % 12);
    wr(in, (int32_t)(g() & 1));
    wr(in, (int32_t)((int)(g() % 8) - 1));
    wr(in, (int32_t)(g() & 1));
    wr(in, (int32_t)(g() % 4));
    wr(in, (int32_t)n_steps);
    wr(in, 1.0 - 1e-5 * u(g));
    wr(in, 1e-6 * u(g));
    wr(in, 0.2 * u(g) - 0.05);
    wr(in, 1e-3 * u(g));
    wr(in, (g() & 1) ? DBL_MAX : u(g));
    for (int i = 0; i < 16; ++i)
      wr(in, (double)(i % 5 == 0));
    for (int k = 0; k < n_steps; ++k) {
      wr(in, (int32_t)(g() % 16 != 0));
      wr(in, u(g));
      const double a = 1e-3 * (u(g) - 0.5), ca = std::cos(a), sa = std::sin(a);
      const double T[16] = {ca, -sa, 0, 1e-3 * (u(g) - 0.5), sa, ca, 0, 1e-3 * (u(g) - 0.5), 0, 0, 1, 0, 0, 0, 0, 1};
      for (int i = 0; i < 16; ++i)
        wr(in, T[i]);
    }
  }
  replay(in, out);
  for (int c = 0; c < n_cases; ++c) {
    const int n = rd<int32_t>(out);
    for (int k = 0; k < n; ++k) {
      const int32_t state = rd<int32_t>(out), converged = rd<int32_t>(out), iterations = rd<int32_t>(out),
                    similar = rd<int32_t>(out);
      rd<double>(out);
      for (int i = 0; i < 16; ++i)
        rd<double>(out);
      const bool last = k == n - 1;
      CHECK(last || state == PCLB200_CONV_NOT_CONVERGED, "case %d step %d: state %d before the last record", c, k, state);
      CHECK(state != PCLB200_CONV_NO_CORRESPONDENCES || (!converged && iterations == k), "case %d step %d", c, k);
      CHECK(state == PCLB200_CONV_NO_CORRESPONDENCES || iterations == k + 1, "case %d step %d: %d iterations", c, k, iterations);
      CHECK(!converged || (state >= PCLB200_CONV_ITERATIONS && state <= PCLB200_CONV_REL_MSE), "case %d step %d", c, k);
      CHECK(similar >= 0 && similar <= iterations, "case %d step %d: similar %d", c, k, similar);
    }
  }
}

int main(int argc, char** argv)
{
  if (argc >= 3) {
    std::ifstream in(argv[1], std::ios::binary);
    std::ofstream out(argv[2], std::ios::binary);
    replay(in, out);
  }
  else
    self_test();
  std::printf("%ld checks, %ld failures\n", g_checks, g_fail);
  if (g_fail)
    return 1;
  std::printf("PASSED\n");
  return 0;
}
