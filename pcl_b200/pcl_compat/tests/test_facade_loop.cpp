// Façade program for the convergence criteria's state across align() calls (runs on the device through
// tests/test_zz_facade_extra_gpu.py, and on the CPU against the oracle-backed test double through
// tests/test_facade_on_oracle.py).  PCL's IterativeClosestPoint creates its DefaultConvergenceCriteria once (icp.h:155);
// the criteria's previous MSE is never reset, so it carries from one align() of the object to the next.
#include <cstdio>

#include <pcl/io/pcd_io.h>
#include <pcl/point_representation.h>
#include <pcl/point_types.h>
#include <pcl/registration/icp.h>

using namespace pcl;

static int g_fail = 0, g_checks = 0;
#define EXPECT_TRUE(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); } } while (0)
#define EXPECT_EQ(a, b) do { ++g_checks; if (!((a) == (b))) { ++g_fail; std::printf("FAIL %s:%d  %s == %s  (%g vs %g)\n", __FILE__, __LINE__, #a, #b, (double)(a), (double)(b)); } } while (0)

int main(int argc, char** argv)
{
  if (argc < 3) { std::fprintf(stderr, "usage: %s bun0.pcd bun4.pcd\n", argv[0]); return 2; }
  PointCloud<PointXYZ> cloud_source, cloud_target;
  if (io::loadPCDFile(argv[1], cloud_source) || io::loadPCDFile(argv[2], cloud_target)) return 2;

  {  // The criteria object outlives one align() (icp.h:155) and its previous MSE is never reset
     // (default_convergence_criteria.h:283, impl/…criteria.hpp:137): a second align() of the same object compares its
     // first iteration with the last MSE the first align recorded.  Every pair lies inside the gate, so every MSE lies in
     // [0, gate^2]; with an absolute threshold of 1 the first align stops at iteration 2 (ABS_MSE) and records only
     // iteration 1's MSE, and the second align, from the first one's result, stops at its iteration 1.  A new object
     // compares iteration 1 with DBL_MAX and stops at iteration 2.  A relative threshold of 0.9 gives the same stops as
     // long as no MSE falls to a tenth of the one before.  Both the fused device loop and the staged loop (forced by a
     // point representation; a uniform rescale by 2 doubles every distance, so the gate doubles too) keep the value.
    using Criteria = registration::DefaultConvergenceCriteria<float>;
    DefaultPointRepresentation<PointXYZ> rep2;
    const float a2[3] = {2.f, 2.f, 2.f};
    rep2.setRescaleValues(a2);
    for (int staged = 0; staged < 2; ++staged)
      for (int relative = 0; relative < 2; ++relative) {
        const int failed_before = g_fail;
        auto make = [&](IterativeClosestPoint<PointXYZ, PointXYZ>& reg) {
          reg.setInputSource(cloud_source.makeShared());
          reg.setInputTarget(cloud_target.makeShared());
          reg.setMaximumIterations(50);
          reg.setMaxCorrespondenceDistance(staged ? 0.1 : 0.05);
          if (staged) reg.setPointRepresentation(rep2.makeShared());
          if (relative) {
            reg.getConvergeCriteria()->setAbsoluteMSE(0.0);
            reg.setEuclideanFitnessEpsilon(0.9);
          }
          else
            reg.getConvergeCriteria()->setAbsoluteMSE(1.0);
        };
        const Criteria::ConvergenceState want = relative ? Criteria::CONVERGENCE_CRITERIA_REL_MSE : Criteria::CONVERGENCE_CRITERIA_ABS_MSE;
        IterativeClosestPoint<PointXYZ, PointXYZ> reg, fresh;
        make(reg);
        make(fresh);
        PointCloud<PointXYZ> out;
        reg.align(out);
        EXPECT_EQ(reg.getNumberOfIterations(), 2);
        EXPECT_EQ(reg.getConvergeCriteria()->getConvergenceState(), want);
        const Eigen::Matrix4f first = reg.getFinalTransformation();
        reg.align(out, first);
        EXPECT_EQ(reg.getNumberOfIterations(), 1);
        EXPECT_EQ(reg.getConvergeCriteria()->getConvergenceState(), want);
        EXPECT_TRUE(reg.hasConverged());
        fresh.align(out, first);
        EXPECT_EQ(fresh.getNumberOfIterations(), 2);
        EXPECT_EQ(fresh.getConvergeCriteria()->getConvergenceState(), want);
        if (g_fail > failed_before) std::printf("carry-over: staged %d relative %d\n", staged, relative);
      }
  }

  std::printf("%d checks, %d failures\n%s\n", g_checks, g_fail, g_fail ? "FAILED" : "PASSED");
  return g_fail ? 1 : 0;
}
