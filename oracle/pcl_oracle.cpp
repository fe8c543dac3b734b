// pcl_oracle.cpp — CPU ORACLE. TEST INFRASTRUCTURE ONLY.
//
// A CPU restatement of PCL's ICP registration hot path (PCL 1.15.1.99), written from the
// behaviour of the reference sources cited beside every function (paths relative to the PCL
// source root).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may load this library; the product (pcl_b200/) never links, imports or
// calls it.  Parity is PINNED: tests/test_oracle_golden.py checks this file against the
// reference's own golden vectors (397 + 53 correspondence pairs, 3283 FLANN radius lists, the
// 10-point k-NN known answer, the bun0->bun4 ICP matrix, VoxelGrid 103/14/100, the bun0 normal).
//
// Third-party arithmetic the reference delegates to and that is NOT under the PCL tree
// (restated here from the published algorithms, anchored on PCL's call sites and tests):
//   * FLANN >= 1.9.1 (KDTreeSingleIndex, L2_Simple, checks=-1, eps=0 => EXACT search):
//       call sites kdtree/include/pcl/kdtree/impl/kdtree_flann.hpp:131-135,154,291.
//       Because the search is exact, any exact k-NN with the same distance arithmetic gives
//       the same result multiset; only the order of exactly-tied distances is FLANN-traversal
//       specific.  Canonical rules used by oracle AND device code:
//         d2 = ((dx*dx) + dy*dy) + dz*dz in fp32, round-to-nearest, NO fma contraction
//         ties broken by the smaller ORIGINAL cloud index
//         radius search keeps d2 < r2 (strict; FLANN RadiusResultSet::addPoint, same rule as
//         PCL's own nanoflann adaptor search/include/pcl/search/kdtree_nanoflann.h:255)
//   * Eigen >= 3.3: umeyama (restated in-tree at common/include/pcl/common/impl/eigen.hpp:675-734),
//       JacobiSVD<3x3> (here: one-sided Jacobi), Matrix<double,6,6>::inverse (here: partial-pivot
//       Gaussian elimination).
//   * Boost spreadsort in VoxelGrid (any key sort gives the same runs; here a STABLE sort so
//       the within-voxel summation order is defined: ascending input index).
//
// Build: see oracle/Makefile (g++ -O3 -ffp-contract=off -fopenmp).  -ffp-contract=off matters:
// the canonical fp32 distance must not be fused.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_API extern "C" __attribute__((visibility("default")))

namespace {

// ------------------------------------------------------------------------------------------
// canonical fp32 squared distance — flann::L2_Simple<float> accumulate loop
// (result += diff*diff over x,y,z), as bound at kdtree/include/pcl/kdtree/kdtree_flann.h:131
// ------------------------------------------------------------------------------------------
static inline float dist2(const float* a, const float* b)
{
  float dx = a[0] - b[0];
  float r = dx * dx;
  float dy = a[1] - b[1];
  r = r + dy * dy;
  float dz = a[2] - b[2];
  r = r + dz * dz;
  return r;
}

static inline bool finite3(const float* p)
{
  return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]);
}

// lower bound of dist2(q, p) for every p inside [lo,hi]; same operation order as dist2 so that
// (by monotonicity of round-to-nearest) bound <= dist2 holds in fp32, not just in the reals.
static inline float box_dist2(const float* q, const float* lo, const float* hi)
{
  float dx = std::max(std::max(lo[0] - q[0], q[0] - hi[0]), 0.0f);
  float r = dx * dx;
  float dy = std::max(std::max(lo[1] - q[1], q[1] - hi[1]), 0.0f);
  r = r + dy * dy;
  float dz = std::max(std::max(lo[2] - q[2], q[2] - hi[2]), 0.0f);
  r = r + dz * dz;
  return r;
}

struct Cand {
  float d;
  int32_t i;
};
static inline bool cand_less(const Cand& a, const Cand& b)
{
  return a.d < b.d || (a.d == b.d && a.i < b.i);
}

// ------------------------------------------------------------------------------------------
// Exact kd-tree, <= 15 points per leaf (KDTreeSingleIndexParams(15), kdtree_flann.hpp:131-134),
// points reordered into leaf order, tight boxes on every node.
// Index semantics follow KdTreeFLANN::convertCloudToArray (kdtree_flann.hpp:429-498):
// non-finite points are dropped and `orig` plays the role of index_mapping_.
// ------------------------------------------------------------------------------------------
struct KdNode {
  float lo[3], hi[3];
  int32_t left, right;  // children (internal) or -1
  int32_t begin, end;   // point range (leaf)
};

struct KdTree {
  std::vector<float> pts;     // n*3, leaf order
  std::vector<int32_t> orig;  // n, original cloud index of pts[i]
  std::vector<KdNode> nodes;
  size_t n = 0;
};


static int32_t kd_build_rec(KdTree& t, std::vector<int32_t>& perm, std::vector<float>& src, int b,
                            int e)
{
  // perm[b..e) index into src (xyz triples)
  KdNode node;
  for (int d = 0; d < 3; ++d) {
    node.lo[d] = FLT_MAX;
    node.hi[d] = -FLT_MAX;
  }
  for (int i = b; i < e; ++i)
    for (int d = 0; d < 3; ++d) {
      float v = src[3 * (size_t)perm[i] + d];
      node.lo[d] = std::min(node.lo[d], v);
      node.hi[d] = std::max(node.hi[d], v);
    }
  node.left = node.right = -1;
  node.begin = b;
  node.end = e;
  int32_t id = (int32_t)t.nodes.size();
  t.nodes.push_back(node);
  if (e - b <= 15)
    return id;
  int dim = 0;
  float span = node.hi[0] - node.lo[0];
  for (int d = 1; d < 3; ++d)
    if (node.hi[d] - node.lo[d] > span) {
      span = node.hi[d] - node.lo[d];
      dim = d;
    }
  float cut = 0.5f * (node.lo[dim] + node.hi[dim]);
  auto mid_it = std::partition(perm.begin() + b, perm.begin() + e,
                               [&](int32_t p) { return src[3 * (size_t)p + dim] < cut; });
  int mid = (int)(mid_it - perm.begin());
  if (mid == b || mid == e) {  // degenerate (duplicates): split by count
    mid = b + (e - b) / 2;
    std::nth_element(perm.begin() + b, perm.begin() + mid, perm.begin() + e,
                     [&](int32_t x, int32_t y) {
                       float vx = src[3 * (size_t)x + dim], vy = src[3 * (size_t)y + dim];
                       return vx < vy || (vx == vy && x < y);
                     });
  }
  int32_t l = kd_build_rec(t, perm, src, b, mid);
  int32_t r = kd_build_rec(t, perm, src, mid, e);
  t.nodes[id].left = l;
  t.nodes[id].right = r;
  return id;
}

struct KnnSet {  // ascending (d, i), capacity k
  Cand* c;
  int k;
  int n;
  inline float worst() const { return n < k ? FLT_MAX : c[k - 1].d; }
  inline bool full() const { return n >= k; }
  inline void offer(Cand x)
  {
    if (n == k) {
      if (!cand_less(x, c[k - 1]))
        return;
      --n;
    }
    int j = n++;
    while (j > 0 && cand_less(x, c[j - 1])) {
      c[j] = c[j - 1];
      --j;
    }
    c[j] = x;
  }
};

static void kd_knn_rec(const KdTree& t, int32_t id, const float* q, KnnSet& rs)
{
  const KdNode& nd = t.nodes[id];
  if (nd.left < 0) {
    for (int i = nd.begin; i < nd.end; ++i) {
      Cand c{dist2(q, &t.pts[3 * (size_t)i]), t.orig[i]};
      rs.offer(c);
    }
    return;
  }
  const KdNode& L = t.nodes[nd.left];
  const KdNode& R = t.nodes[nd.right];
  float dl = box_dist2(q, L.lo, L.hi), dr = box_dist2(q, R.lo, R.hi);
  int32_t first = nd.left, second = nd.right;
  if (dr < dl) {
    std::swap(first, second);
    std::swap(dl, dr);
  }
  // prune only when strictly worse than the current k-th: an equal-distance point with a
  // smaller index must still be able to displace it (canonical tie rule).
  if (!(rs.full() && dl > rs.worst()))
    kd_knn_rec(t, first, q, rs);
  if (!(rs.full() && dr > rs.worst()))
    kd_knn_rec(t, second, q, rs);
}

static void kd_radius_rec(const KdTree& t, int32_t id, const float* q, float r2,
                          std::vector<Cand>& out)
{
  const KdNode& nd = t.nodes[id];
  if (box_dist2(q, nd.lo, nd.hi) >= r2)
    return;
  if (nd.left < 0) {
    for (int i = nd.begin; i < nd.end; ++i) {
      float d = dist2(q, &t.pts[3 * (size_t)i]);
      if (d < r2)
        out.push_back(Cand{d, t.orig[i]});
    }
    return;
  }
  kd_radius_rec(t, nd.left, q, r2, out);
  kd_radius_rec(t, nd.right, q, r2, out);
}

// ------------------------------------------------------------------------------------------
// small dense linear algebra (the reference delegates these to Eigen)
// ------------------------------------------------------------------------------------------
template <typename S>
static S det3(const S m[9])
{
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) +
         m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// One-sided (Hestenes) Jacobi SVD of a row-major 3x3: A = U diag(s) V^T, s descending.
template <typename S>
static void svd3(const S Ain[9], S U[9], S s[3], S V[9])
{
  S A[9];
  for (int i = 0; i < 9; ++i)
    A[i] = Ain[i];
  for (int i = 0; i < 9; ++i)
    V[i] = (i % 4 == 0) ? S(1) : S(0);
  const S eps = std::numeric_limits<S>::epsilon();
  for (int sweep = 0; sweep < 60; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        S alpha = 0, beta = 0, gamma = 0;
        for (int i = 0; i < 3; ++i) {
          alpha += A[3 * i + p] * A[3 * i + p];
          beta += A[3 * i + q] * A[3 * i + q];
          gamma += A[3 * i + p] * A[3 * i + q];
        }
        if (gamma == S(0) || std::abs(gamma) <= eps * std::sqrt(alpha * beta))
          continue;
        rotated = true;
        S zeta = (beta - alpha) / (S(2) * gamma);
        S tt = (zeta >= 0 ? S(1) : S(-1)) / (std::abs(zeta) + std::sqrt(S(1) + zeta * zeta));
        S c = S(1) / std::sqrt(S(1) + tt * tt), sn = c * tt;
        for (int i = 0; i < 3; ++i) {
          S ap = A[3 * i + p], aq = A[3 * i + q];
          A[3 * i + p] = c * ap - sn * aq;
          A[3 * i + q] = sn * ap + c * aq;
          S vp = V[3 * i + p], vq = V[3 * i + q];
          V[3 * i + p] = c * vp - sn * vq;
          V[3 * i + q] = sn * vp + c * vq;
        }
      }
    if (!rotated)
      break;
  }
  S nrm[3];
  for (int j = 0; j < 3; ++j)
    nrm[j] = std::sqrt(A[j] * A[j] + A[3 + j] * A[3 + j] + A[6 + j] * A[6 + j]);
  int ord[3] = {0, 1, 2};
  std::sort(ord, ord + 3, [&](int a, int b) { return nrm[a] > nrm[b]; });
  S Vs[9];
  for (int j = 0; j < 3; ++j) {
    s[j] = nrm[ord[j]];
    for (int i = 0; i < 3; ++i) {
      Vs[3 * i + j] = V[3 * i + ord[j]];
      U[3 * i + j] = (s[j] > S(0)) ? A[3 * i + ord[j]] / s[j] : S(0);
    }
  }
  for (int i = 0; i < 9; ++i)
    V[i] = Vs[i];
  // complete U for (near-)rank-deficient input so that U stays orthogonal
  const S tiny = s[0] * eps * S(8);
  if (s[0] <= S(0)) {
    for (int i = 0; i < 9; ++i)
      U[i] = (i % 4 == 0) ? S(1) : S(0);
    return;
  }
  if (s[1] <= tiny) {  // rank 1: any unit vector orthogonal to u0
    S u0[3] = {U[0], U[3], U[6]};
    int m = 0;
    if (std::abs(u0[1]) < std::abs(u0[m]))
      m = 1;
    if (std::abs(u0[2]) < std::abs(u0[m]))
      m = 2;
    S e[3] = {0, 0, 0};
    e[m] = 1;
    S w[3] = {u0[1] * e[2] - u0[2] * e[1], u0[2] * e[0] - u0[0] * e[2], u0[0] * e[1] - u0[1] * e[0]};
    S wn = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    for (int i = 0; i < 3; ++i)
      U[3 * i + 1] = w[i] / wn;
  }
  if (s[2] <= tiny) {  // u2 = u0 x u1
    S a[3] = {U[0], U[3], U[6]}, b[3] = {U[1], U[4], U[7]};
    U[2] = a[1] * b[2] - a[2] * b[1];
    U[5] = a[2] * b[0] - a[0] * b[2];
    U[8] = a[0] * b[1] - a[1] * b[0];
  }
}

// x = A^-1 b for a 6x6 (row-major), partial pivoting.  Stands in for
// `ATA.inverse() * ATb` (transformation_estimation_point_to_plane_lls.hpp:264).
static bool solve6(const double Ain[36], const double bin[6], double x[6])
{
  double A[6][7];
  for (int i = 0; i < 6; ++i) {
    for (int j = 0; j < 6; ++j)
      A[i][j] = Ain[6 * i + j];
    A[i][6] = bin[i];
  }
  for (int c = 0; c < 6; ++c) {
    int piv = c;
    for (int r = c + 1; r < 6; ++r)
      if (std::abs(A[r][c]) > std::abs(A[piv][c]))
        piv = r;
    if (A[piv][c] == 0.0)
      return false;
    if (piv != c)
      for (int j = 0; j < 7; ++j)
        std::swap(A[piv][j], A[c][j]);
    for (int r = c + 1; r < 6; ++r) {
      double f = A[r][c] / A[c][c];
      for (int j = c; j < 7; ++j)
        A[r][j] -= f * A[c][j];
    }
  }
  for (int r = 5; r >= 0; --r) {
    double acc = A[r][6];
    for (int j = r + 1; j < 6; ++j)
      acc -= A[r][j] * x[j];
    x[r] = acc / A[r][r];
  }
  return true;
}

// ------------------------------------------------------------------------------------------
// TransformationEstimationSVD (use_umeyama_ = true) —
// registration/include/pcl/registration/impl/transformation_estimation_svd.hpp:137-155 gathers
// the pairs, pcl::umeyama(src, dst, false) (common/include/pcl/common/impl/eigen.hpp:675-734):
// means, demean, sigma = 1/n * dst_d * src_d^T, SVD, S = diag(1,1,sign), R = U S V^T,
// t = mean_dst - R mean_src.   T is row-major 4x4 of Scalar S.
// ------------------------------------------------------------------------------------------
template <typename S>
static void umeyama(const float* src, size_t ss, const float* tgt, size_t ts, const int32_t* qi,
                    const int32_t* mi, size_t n, S T[16])
{
  const S one_over_n = S(1) / static_cast<S>(n);
  S ms[3] = {0, 0, 0}, md[3] = {0, 0, 0};
  for (size_t i = 0; i < n; ++i) {
    const float* p = src + ss * (size_t)(qi ? qi[i] : (int32_t)i);
    const float* q = tgt + ts * (size_t)(mi ? mi[i] : (int32_t)i);
    for (int d = 0; d < 3; ++d) {
      ms[d] += static_cast<S>(p[d]);
      md[d] += static_cast<S>(q[d]);
    }
  }
  for (int d = 0; d < 3; ++d) {
    ms[d] *= one_over_n;
    md[d] *= one_over_n;
  }
  S sig[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (size_t i = 0; i < n; ++i) {
    const float* p = src + ss * (size_t)(qi ? qi[i] : (int32_t)i);
    const float* q = tgt + ts * (size_t)(mi ? mi[i] : (int32_t)i);
    S pd[3], qd[3];
    for (int d = 0; d < 3; ++d) {
      pd[d] = static_cast<S>(p[d]) - ms[d];
      qd[d] = static_cast<S>(q[d]) - md[d];
    }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        sig[3 * r + c] += qd[r] * pd[c];
  }
  for (int i = 0; i < 9; ++i)
    sig[i] *= one_over_n;
  S U[9], sv[3], V[9];
  svd3<S>(sig, U, sv, V);
  S Sd[3] = {1, 1, 1};
  if (det3<S>(U) * det3<S>(V) < S(0))
    Sd[2] = S(-1);
  S R[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      S acc = 0;
      for (int k = 0; k < 3; ++k)
        acc += U[3 * r + k] * Sd[k] * V[3 * c + k];
      R[3 * r + c] = acc;
    }
  for (int i = 0; i < 16; ++i)
    T[i] = (i % 5 == 0) ? S(1) : S(0);
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c)
      T[4 * r + c] = R[3 * r + c];
    T[4 * r + 3] = md[r] - (R[3 * r] * ms[0] + R[3 * r + 1] * ms[1] + R[3 * r + 2] * ms[2]);
  }
}

// ------------------------------------------------------------------------------------------
// TransformationEstimationPointToPlaneLLS —
// registration/include/pcl/registration/impl/transformation_estimation_point_to_plane_lls.hpp
// :166-268 (accumulate; a,b,c and d are FLOAT expressions widened to double at :202-204,235)
// and :132-163 (constructTransformationMatrix, R = Rz(gamma) Ry(beta) Rx(alpha)).
// tn = target normals (float pointer to nx of point 0, same stride ts as tgt).
// ------------------------------------------------------------------------------------------
template <typename S>
static bool p2plane_lls(const float* src, size_t ss, const float* tgt, const float* tn, size_t ts,
                        const int32_t* qi, const int32_t* mi, size_t n, S T[16])
{
  double ATA[36], ATb[6];
  std::fill(ATA, ATA + 36, 0.0);
  std::fill(ATb, ATb + 6, 0.0);
  for (size_t i = 0; i < n; ++i) {
    size_t si = (size_t)(qi ? qi[i] : (int32_t)i), ti = (size_t)(mi ? mi[i] : (int32_t)i);
    const float* s = src + ss * si;
    const float* t = tgt + ts * ti;
    const float* nn = tn + ts * ti;
    if (!finite3(s) || !finite3(t) || !finite3(nn))
      continue;
    const float sx = s[0], sy = s[1], sz = s[2], dx = t[0], dy = t[1], dz = t[2];
    const float nx = nn[0], ny = nn[1], nz = nn[2];
    double a = nz * sy - ny * sz;
    double b = nx * sz - nz * sx;
    double c = ny * sx - nx * sy;
    ATA[0] += a * a;
    ATA[1] += a * b;
    ATA[2] += a * c;
    ATA[3] += a * nx;
    ATA[4] += a * ny;
    ATA[5] += a * nz;
    ATA[7] += b * b;
    ATA[8] += b * c;
    ATA[9] += b * nx;
    ATA[10] += b * ny;
    ATA[11] += b * nz;
    ATA[14] += c * c;
    ATA[15] += c * nx;
    ATA[16] += c * ny;
    ATA[17] += c * nz;
    ATA[21] += nx * nx;
    ATA[22] += nx * ny;
    ATA[23] += nx * nz;
    ATA[28] += ny * ny;
    ATA[29] += ny * nz;
    ATA[35] += nz * nz;
    double d = nx * dx + ny * dy + nz * dz - nx * sx - ny * sy - nz * sz;
    ATb[0] += a * d;
    ATb[1] += b * d;
    ATb[2] += c * d;
    ATb[3] += nx * d;
    ATb[4] += ny * d;
    ATb[5] += nz * d;
  }
  for (int r = 1; r < 6; ++r)
    for (int c = 0; c < r; ++c)
      ATA[6 * r + c] = ATA[6 * c + r];
  double x[6];
  bool ok = solve6(ATA, ATb, x);
  if (!ok)
    for (int i = 0; i < 6; ++i)
      x[i] = std::numeric_limits<double>::quiet_NaN();
  const double alpha = x[0], beta = x[1], gamma = x[2];
  for (int i = 0; i < 16; ++i)
    T[i] = S(0);
  T[0] = static_cast<S>(std::cos(gamma) * std::cos(beta));
  T[1] = static_cast<S>(-std::sin(gamma) * std::cos(alpha) +
                        std::cos(gamma) * std::sin(beta) * std::sin(alpha));
  T[2] = static_cast<S>(std::sin(gamma) * std::sin(alpha) +
                        std::cos(gamma) * std::sin(beta) * std::cos(alpha));
  T[4] = static_cast<S>(std::sin(gamma) * std::cos(beta));
  T[5] = static_cast<S>(std::cos(gamma) * std::cos(alpha) +
                        std::sin(gamma) * std::sin(beta) * std::sin(alpha));
  T[6] = static_cast<S>(-std::cos(gamma) * std::sin(alpha) +
                        std::sin(gamma) * std::sin(beta) * std::cos(alpha));
  T[8] = static_cast<S>(-std::sin(beta));
  T[9] = static_cast<S>(std::cos(beta) * std::sin(alpha));
  T[10] = static_cast<S>(std::cos(beta) * std::cos(alpha));
  T[3] = static_cast<S>(x[3]);
  T[7] = static_cast<S>(x[4]);
  T[11] = static_cast<S>(x[5]);
  T[15] = S(1);
  return ok;
}

// ------------------------------------------------------------------------------------------
// TransformationEstimationSymmetricPointToPlaneLLS (SURVEY.md §8f #2) —
// registration/include/pcl/registration/impl/transformation_estimation_symmetric_point_to_plane_lls.hpp
// :150-200 (v = [(p+q) x n, n], n = n1 +/- n2, rank-1 updates and v*((q-p).n) accumulated in Scalar, LDLT solve)
// and :128-147 (T = Rz Ry Rx * translation * Rz Ry Rx).  sn / tn = first nx of source / target normals.
// ------------------------------------------------------------------------------------------
template <typename S>
static bool sym_p2plane_lls(const float* src, const float* sn, size_t ss, const float* tgt, const float* tn, size_t ts,
                            const int32_t* qi, const int32_t* mi, size_t n, bool enforce_same_direction, S T[16])
{
  S ATA[36], ATb[6];
  for (int i = 0; i < 36; ++i) ATA[i] = S(0);
  for (int i = 0; i < 6; ++i) ATb[i] = S(0);
  for (size_t i = 0; i < n; ++i) {
    size_t si = (size_t)(qi ? qi[i] : (int32_t)i), ti = (size_t)(mi ? mi[i] : (int32_t)i);
    const float* pf = src + ss * si;
    const float* qf = tgt + ts * ti;
    const float* n1f = sn + ss * si;
    const float* n2f = tn + ts * ti;
    S p[3], q[3], n1[3], n2[3], nn[3];
    for (int d = 0; d < 3; ++d) { p[d] = pf[d]; q[d] = qf[d]; n1[d] = n1f[d]; n2[d] = n2f[d]; }
    const bool same = !enforce_same_direction || (n1[0] * n2[0] + n1[1] * n2[1] + n1[2] * n2[2]) >= S(0);
    for (int d = 0; d < 3; ++d) nn[d] = same ? n1[d] + n2[d] : n1[d] - n2[d];
    if (!std::isfinite(p[0] + p[1] + p[2]) || !std::isfinite(q[0] + q[1] + q[2]) || !std::isfinite(nn[0] + nn[1] + nn[2]))
      continue;
    const S s3[3] = {p[0] + q[0], p[1] + q[1], p[2] + q[2]};
    S v[6] = {s3[1] * nn[2] - s3[2] * nn[1], s3[2] * nn[0] - s3[0] * nn[2], s3[0] * nn[1] - s3[1] * nn[0], nn[0], nn[1], nn[2]};
    for (int r = 0; r < 6; ++r)
      for (int c = r; c < 6; ++c)
        ATA[6 * r + c] += v[r] * v[c];
    const S b = (q[0] - p[0]) * nn[0] + (q[1] - p[1]) * nn[1] + (q[2] - p[2]) * nn[2];
    for (int r = 0; r < 6; ++r)
      ATb[r] += v[r] * b;
  }
  double A[36], B[6], x[6];
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c)
      A[6 * r + c] = static_cast<double>(c >= r ? ATA[6 * r + c] : ATA[6 * c + r]);
  for (int r = 0; r < 6; ++r)
    B[r] = static_cast<double>(ATb[r]);
  bool ok = solve6(A, B, x);
  if (!ok)
    for (int i = 0; i < 6; ++i) x[i] = std::numeric_limits<double>::quiet_NaN();
  const S al = static_cast<S>(x[0]), be = static_cast<S>(x[1]), ga = static_cast<S>(x[2]);
  const S ca = std::cos(al), sa = std::sin(al), cb = std::cos(be), sb = std::sin(be), cg = std::cos(ga), sg = std::sin(ga);
  // R = Rz(ga) Ry(be) Rx(al)
  const S Rm[9] = {cg * cb, cg * sb * sa - sg * ca, cg * sb * ca + sg * sa,
                   sg * cb, sg * sb * sa + cg * ca, sg * sb * ca - cg * sa,
                   -sb,     cb * sa,                cb * ca};
  const S tr[3] = {static_cast<S>(x[3]), static_cast<S>(x[4]), static_cast<S>(x[5])};
  // T = [R | 0] * [I | t] * [R | 0] = [R R | R t]
  for (int i = 0; i < 16; ++i) T[i] = S(0);
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c)
      T[4 * r + c] = Rm[3 * r] * Rm[c] + Rm[3 * r + 1] * Rm[3 + c] + Rm[3 * r + 2] * Rm[6 + c];
    T[4 * r + 3] = Rm[3 * r] * tr[0] + Rm[3 * r + 1] * tr[1] + Rm[3 * r + 2] * tr[2];
  }
  T[15] = S(1);
  return ok;
}

// ------------------------------------------------------------------------------------------
// point transforms
//   mode 0: IterativeClosestPoint::transformCloud (registration/.../impl/icp.hpp:49-111):
//           tr = transform.cast<float>(); pt_t = tr * (x,y,z,1)  -> ((c0*x + c1*y) + c2*z) + c3
//           (Eigen coefficient-based 4x4 * 4x1 product), normals nt_t = rot * nt likewise;
//           non-finite points (and non-finite normals) are left untouched.
//   mode 1: pcl::transformPointCloud[WithNormals] (common/.../impl/transforms.hpp:67-133, SSE2
//           Transformer<float>): se3 = c0*x + (c1*y + (c2*z + c3)), so3 = c0*x + (c1*y + c2*z);
//           Transformer<double> (:135-181): ((c3 + x*c0) + y*c1) + z*c2 in double, then -> float.
// T is row-major 4x4 of Scalar S; for mode 0 it is first cast to float like the reference.
// ------------------------------------------------------------------------------------------
template <typename S>
static void transform_points(float* pts, size_t n, size_t stride, int normal_off, const S T[16],
                             int mode)
{
  if (mode == 0) {
    float m[16];
    for (int i = 0; i < 16; ++i)
      m[i] = static_cast<float>(T[i]);
    for (size_t i = 0; i < n; ++i) {
      float* p = pts + stride * i;
      if (!finite3(p))
        continue;
      float x = p[0], y = p[1], z = p[2];
      p[0] = ((m[0] * x + m[1] * y) + m[2] * z) + m[3];
      p[1] = ((m[4] * x + m[5] * y) + m[6] * z) + m[7];
      p[2] = ((m[8] * x + m[9] * y) + m[10] * z) + m[11];
      if (normal_off >= 0) {
        float* nn = p + normal_off;
        if (!finite3(nn))
          continue;
        float a = nn[0], b = nn[1], c = nn[2];
        nn[0] = (m[0] * a + m[1] * b) + m[2] * c;
        nn[1] = (m[4] * a + m[5] * b) + m[6] * c;
        nn[2] = (m[8] * a + m[9] * b) + m[10] * c;
      }
    }
    return;
  }
  for (size_t i = 0; i < n; ++i) {
    float* p = pts + stride * i;
    // transformPointCloud on a dense cloud transforms unconditionally; on a non-dense cloud it
    // skips non-finite points (transforms.hpp:95-110).  Non-finite stays non-finite either way.
    if (!finite3(p))
      continue;
    if (sizeof(S) == sizeof(float)) {
      float x = p[0], y = p[1], z = p[2];
      const float* m = reinterpret_cast<const float*>(T);
      p[0] = m[0] * x + (m[1] * y + (m[2] * z + m[3]));
      p[1] = m[4] * x + (m[5] * y + (m[6] * z + m[7]));
      p[2] = m[8] * x + (m[9] * y + (m[10] * z + m[11]));
      if (normal_off >= 0) {
        float* nn = p + normal_off;
        float a = nn[0], b = nn[1], c = nn[2];
        nn[0] = m[0] * a + (m[1] * b + m[2] * c);
        nn[1] = m[4] * a + (m[5] * b + m[6] * c);
        nn[2] = m[8] * a + (m[9] * b + m[10] * c);
      }
    }
    else {
      const double* m = reinterpret_cast<const double*>(T);
      double x = p[0], y = p[1], z = p[2];
      p[0] = static_cast<float>(((m[3] + x * m[0]) + y * m[1]) + z * m[2]);
      p[1] = static_cast<float>(((m[7] + x * m[4]) + y * m[5]) + z * m[6]);
      p[2] = static_cast<float>(((m[11] + x * m[8]) + y * m[9]) + z * m[10]);
      if (normal_off >= 0) {
        float* nn = p + normal_off;
        double a = nn[0], b = nn[1], c = nn[2];
        nn[0] = static_cast<float>((a * m[0] + b * m[1]) + c * m[2]);
        nn[1] = static_cast<float>((a * m[4] + b * m[5]) + c * m[6]);
        nn[2] = static_cast<float>((a * m[8] + b * m[9]) + c * m[10]);
      }
    }
  }
}

// C = A * B, row-major 4x4 in Scalar S, Eigen coefficient order ((a0*b0 + a1*b1) + a2*b2) + a3*b3
// — `final_transformation_ = transformation_ * final_transformation_` (icp.hpp:223).
template <typename S>
static void mat4_mul(const S A[16], const S B[16], S C[16])
{
  S R[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c)
      R[4 * r + c] = ((A[4 * r] * B[c] + A[4 * r + 1] * B[4 + c]) + A[4 * r + 2] * B[8 + c]) +
                     A[4 * r + 3] * B[12 + c];
  for (int i = 0; i < 16; ++i)
    C[i] = R[i];
}

// ------------------------------------------------------------------------------------------
// DefaultConvergenceCriteria — registration/include/pcl/registration/default_convergence_criteria.h
// :263-321 (state, defaults, calculateMSE) and impl/default_convergence_criteria.hpp:49-140.
// ------------------------------------------------------------------------------------------
enum ConvState {
  NOT_CONVERGED = 0,
  ITERATIONS = 1,
  TRANSFORM = 2,
  ABS_MSE = 3,
  REL_MSE = 4,
  NO_CORRESPONDENCES = 5,
  FAILURE_AFTER_MAX_ITERATIONS = 6
};

template <typename S>
struct Convergence {
  double prev_mse = std::numeric_limits<double>::max();
  double cur_mse = std::numeric_limits<double>::max();
  int max_iterations = 100;
  bool failure_after_max_iter = false;
  double rotation_threshold = 0.99999;
  double translation_threshold = 3e-4 * 3e-4;
  double mse_threshold_relative = 0.00001;
  double mse_threshold_absolute = 1e-12;
  int iterations_similar_transforms = 0;
  int max_iterations_similar_transforms = 0;
  int state = NOT_CONVERGED;

  bool has_converged(int iterations, const S T[16], double mse)
  {
    if (state != NOT_CONVERGED) {
      iterations_similar_transforms = 0;
      state = NOT_CONVERGED;
    }
    bool is_similar = false;
    if (iterations >= max_iterations) {
      if (!failure_after_max_iter) {
        state = ITERATIONS;
        return true;
      }
      state = FAILURE_AFTER_MAX_ITERATIONS;
    }
    // the trace and the squared norm are evaluated in Scalar, then widened (…criteria.hpp:77-81)
    double cos_angle = 0.5 * (T[0] + T[5] + T[10] - 1);
    double translation_sqr = T[3] * T[3] + T[7] * T[7] + T[11] * T[11];
    if (cos_angle >= rotation_threshold && translation_sqr <= translation_threshold) {
      if (iterations_similar_transforms >= max_iterations_similar_transforms) {
        state = TRANSFORM;
        return true;
      }
      is_similar = true;
    }
    cur_mse = mse;
    if (std::abs(cur_mse - prev_mse) < mse_threshold_absolute) {
      if (iterations_similar_transforms >= max_iterations_similar_transforms) {
        state = ABS_MSE;
        return true;
      }
      is_similar = true;
    }
    if (std::abs(cur_mse - prev_mse) / prev_mse < mse_threshold_relative) {
      if (iterations_similar_transforms >= max_iterations_similar_transforms) {
        state = REL_MSE;
        return true;
      }
      is_similar = true;
    }
    if (is_similar)
      ++iterations_similar_transforms;
    else
      iterations_similar_transforms = 0;
    prev_mse = cur_mse;
    return false;
  }
};

// ------------------------------------------------------------------------------------------
// pcl::eigen33 smallest eigenpair — common/include/pcl/common/impl/eigen.hpp:52-66 (computeRoots2),
// :68-133 (computeRoots), :273-288 (getLargest3x3Eigenvector), :293-326 (eigen33), fp32.
// m is a row-major symmetric 3x3.
// ------------------------------------------------------------------------------------------
static void roots2(float b, float c, float roots[3])
{
  roots[0] = 0.0f;
  float d = static_cast<float>(b * b - 4.0 * c);
  if (d < 0.0)
    d = 0.0;
  float sd = std::sqrt(d);
  roots[2] = 0.5f * (b + sd);
  roots[1] = 0.5f * (b - sd);
}

static void roots3(const float m[9], float roots[3])
{
  float c0 = m[0] * m[4] * m[8] + 2.0f * m[1] * m[2] * m[5] - m[0] * m[5] * m[5] -
             m[4] * m[2] * m[2] - m[8] * m[1] * m[1];
  float c1 = m[0] * m[4] - m[1] * m[1] + m[0] * m[8] - m[2] * m[2] + m[4] * m[8] - m[5] * m[5];
  float c2 = m[0] + m[4] + m[8];
  if (std::abs(c0) < std::numeric_limits<float>::epsilon())
    roots2(c2, c1, roots);
  else {
    const float s_inv3 = static_cast<float>(1.0 / 3.0);
    const float s_sqrt3 = std::sqrt(3.0f);
    float c2_over_3 = c2 * s_inv3;
    float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
    if (a_over_3 > 0.0f)
      a_over_3 = 0.0f;
    float half_b = 0.5f * (c0 + c2_over_3 * (2.0f * c2_over_3 * c2_over_3 - c1));
    float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
    if (q > 0.0f)
      q = 0.0f;
    float rho = std::sqrt(-a_over_3);
    float theta = std::atan2(std::sqrt(-q), half_b) * s_inv3;
    float cos_theta = std::cos(theta);
    float sin_theta = std::sin(theta);
    roots[0] = c2_over_3 + 2.0f * rho * cos_theta;
    roots[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
    roots[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
    if (roots[0] >= roots[1])
      std::swap(roots[0], roots[1]);
    if (roots[1] >= roots[2]) {
      std::swap(roots[1], roots[2]);
      if (roots[0] >= roots[1])
        std::swap(roots[0], roots[1]);
    }
    if (roots[0] <= 0)
      roots2(c2, c1, roots);
  }
}

static void largest_eigvec(const float s[9], float v[3])
{
  // rows crossed pairwise, longest wins (first maximum, like Eigen's maxCoeff)
  const float* r0 = s;
  const float* r1 = s + 3;
  const float* r2 = s + 6;
  float c[3][3] = {
      {r0[1] * r1[2] - r0[2] * r1[1], r0[2] * r1[0] - r0[0] * r1[2], r0[0] * r1[1] - r0[1] * r1[0]},
      {r0[1] * r2[2] - r0[2] * r2[1], r0[2] * r2[0] - r0[0] * r2[2], r0[0] * r2[1] - r0[1] * r2[0]},
      {r1[1] * r2[2] - r1[2] * r2[1], r1[2] * r2[0] - r1[0] * r2[2], r1[0] * r2[1] - r1[1] * r2[0]}};
  float len[3];
  for (int i = 0; i < 3; ++i)
    len[i] = std::sqrt(c[i][0] * c[i][0] + c[i][1] * c[i][1] + c[i][2] * c[i][2]);
  int idx = 0;
  if (len[1] > len[idx])
    idx = 1;
  if (len[2] > len[idx])
    idx = 2;
  for (int d = 0; d < 3; ++d)
    v[d] = c[idx][d] / len[idx];
}

static void unit_orthogonal(const float v[3], float o[3])
{
  // Eigen::MatrixBase::unitOrthogonal() for 3-vectors
  auto much_smaller = [](float a, float b) {
    return std::abs(a) <= std::abs(b) * std::numeric_limits<float>::epsilon();
  };
  if (!much_smaller(v[0], v[2]) || !much_smaller(v[1], v[2])) {
    float invnm = 1.0f / std::sqrt(v[0] * v[0] + v[1] * v[1]);
    o[0] = -v[1] * invnm;
    o[1] = v[0] * invnm;
    o[2] = 0.0f;
  }
  else {
    float invnm = 1.0f / std::sqrt(v[1] * v[1] + v[2] * v[2]);
    o[0] = 0.0f;
    o[1] = -v[2] * invnm;
    o[2] = v[1] * invnm;
  }
}

static void eigen33_smallest(const float mat[9], float& eigenvalue, float ev[3])
{
  float scale = 0.0f;
  for (int i = 0; i < 9; ++i)
    scale = std::max(scale, std::abs(mat[i]));
  if (scale <= std::numeric_limits<float>::min())
    scale = 1.0f;
  float s[9];
  for (int i = 0; i < 9; ++i)
    s[i] = mat[i] / scale;
  float roots[3];
  roots3(s, roots);
  eigenvalue = roots[0] * scale;
  if ((roots[1] - roots[0]) > std::numeric_limits<float>::epsilon()) {
    s[0] -= roots[0];
    s[4] -= roots[0];
    s[8] -= roots[0];
    largest_eigvec(s, ev);
  }
  else if ((roots[2] - roots[0]) > std::numeric_limits<float>::epsilon()) {
    s[0] -= roots[2];
    s[4] -= roots[2];
    s[8] -= roots[2];
    float v[3];
    largest_eigvec(s, v);
    unit_orthogonal(v, ev);
  }
  else {
    ev[0] = 1.0f;
    ev[1] = 0.0f;
    ev[2] = 0.0f;
  }
}

// computeMeanAndCovarianceMatrix (common/include/pcl/common/impl/centroid.hpp:578-652, Scalar =
// float) + solvePlaneParameters (features/include/pcl/features/impl/feature.hpp:65-92).
// Returns false when < 3 usable neighbours (NormalEstimation::computePointNormal,
// features/include/pcl/features/normal_3d.h:308-322).
static bool point_normal(const float* cloud, size_t stride, bool dense, const int32_t* idx, size_t k,
                         float out[4])
{
  const float qnan = std::numeric_limits<float>::quiet_NaN();
  out[0] = out[1] = out[2] = out[3] = qnan;
  if (k < 3)
    return false;
  float K[3] = {0, 0, 0};
  for (size_t i = 0; i < k; ++i) {
    const float* p = cloud + stride * (size_t)idx[i];
    if (finite3(p)) {
      K[0] = p[0];
      K[1] = p[1];
      K[2] = p[2];
      break;
    }
  }
  float accu[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  size_t count = 0;
  for (size_t i = 0; i < k; ++i) {
    const float* p = cloud + stride * (size_t)idx[i];
    if (!dense && !finite3(p))
      continue;
    ++count;
    float x = p[0] - K[0], y = p[1] - K[1], z = p[2] - K[2];
    accu[0] += x * x;
    accu[1] += x * y;
    accu[2] += x * z;
    accu[3] += y * y;
    accu[4] += y * z;
    accu[5] += z * z;
    accu[6] += x;
    accu[7] += y;
    accu[8] += z;
  }
  if (count == 0)
    return false;
  float fc = static_cast<float>(count);
  for (int i = 0; i < 9; ++i)
    accu[i] /= fc;
  float cov[9];
  cov[0] = accu[0] - accu[6] * accu[6];
  cov[1] = accu[1] - accu[6] * accu[7];
  cov[2] = accu[2] - accu[6] * accu[8];
  cov[4] = accu[3] - accu[7] * accu[7];
  cov[5] = accu[4] - accu[7] * accu[8];
  cov[8] = accu[5] - accu[8] * accu[8];
  cov[3] = cov[1];
  cov[6] = cov[2];
  cov[7] = cov[5];
  float ev, n[3];
  eigen33_smallest(cov, ev, n);
  out[0] = n[0];
  out[1] = n[1];
  out[2] = n[2];
  float eig_sum = cov[0] + cov[4] + cov[8];
  out[3] = (eig_sum != 0) ? std::abs(ev / eig_sum) : 0.0f;
  return true;
}

// flipNormalTowardsViewpoint — features/include/pcl/features/normal_3d.h:169-188
static inline void flip_to_viewpoint(const float* p, const float vp[3], float n[3])
{
  float vx = vp[0] - p[0], vy = vp[1] - p[1], vz = vp[2] - p[2];
  float cos_theta = (vx * n[0] + vy * n[1] + vz * n[2]);
  if (cos_theta < 0) {
    n[0] *= -1;
    n[1] *= -1;
    n[2] *= -1;
  }
}

}  // namespace

// ==========================================================================================
// C entry points (ctypes-friendly).  Strides are in FLOATS.
// ==========================================================================================

struct orc_corr {
  int32_t index_query;
  int32_t index_match;
  float distance;
};  // pcl::Correspondence, common/include/pcl/correspondence.h:60-71

// ---- index ------------------------------------------------------------------------------
// KdTreeFLANN::setInputCloud (+indices) — kdtree_flann.hpp:100-136, 429-498
ORC_API void* orc_index_build(const float* pts, size_t n, size_t stride, const int32_t* subset,
                              size_t n_subset)
{
  KdTree* t = new KdTree();
  std::vector<float> src;
  size_t cnt = subset ? n_subset : n;
  src.reserve(3 * cnt);
  t->orig.reserve(cnt);
  std::vector<int32_t> orig0;
  orig0.reserve(cnt);
  for (size_t i = 0; i < cnt; ++i) {
    size_t ci = subset ? (size_t)subset[i] : i;
    const float* p = pts + stride * ci;
    if (!finite3(p))
      continue;
    src.push_back(p[0]);
    src.push_back(p[1]);
    src.push_back(p[2]);
    orig0.push_back((int32_t)ci);
  }
  t->n = orig0.size();
  if (t->n == 0)
    return t;
  std::vector<int32_t> perm(t->n);
  std::iota(perm.begin(), perm.end(), 0);
  t->nodes.reserve(t->n / 4 + 16);
  kd_build_rec(*t, perm, src, 0, (int)t->n);
  t->pts.resize(3 * t->n);
  t->orig.resize(t->n);
  for (size_t i = 0; i < t->n; ++i) {
    std::memcpy(&t->pts[3 * i], &src[3 * (size_t)perm[i]], 3 * sizeof(float));
    t->orig[i] = orig0[perm[i]];
  }
  return t;
}
ORC_API void orc_index_free(void* h) { delete static_cast<KdTree*>(h); }
ORC_API size_t orc_index_size(void* h) { return static_cast<KdTree*>(h)->n; }

// ---- k-NN -------------------------------------------------------------------------------
// KdTreeFLANN::nearestKSearch — kdtree_flann.hpp:234-274: k clamped to #valid points, results
// ascending by distance, indices mapped back to the original cloud.  Returns the clamped k;
// outputs are written with row pitch `k` (the REQUESTED k); unused slots = (-1, +inf).
ORC_API int orc_knn(void* h, const float* q, size_t nq, size_t qstride, int k, int32_t* out_idx,
                    float* out_d2, int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h);
  int keff = (int)std::min<size_t>((size_t)std::max(k, 0), t.n);
  if (k <= 0)
    return 0;
#pragma omp parallel num_threads(nthreads > 0 ? nthreads : 1)
  {
    std::vector<Cand> buf((size_t)std::max(keff, 1));
#pragma omp for schedule(dynamic, 1024)
    for (long long i = 0; i < (long long)nq; ++i) {
      KnnSet rs{buf.data(), keff, 0};
      if (keff > 0)
        kd_knn_rec(t, 0, q + qstride * (size_t)i, rs);
      for (int j = 0; j < k; ++j) {
        out_idx[(size_t)i * k + j] = j < rs.n ? rs.c[j].i : -1;
        out_d2[(size_t)i * k + j] = j < rs.n ? rs.c[j].d : std::numeric_limits<float>::infinity();
      }
    }
  }
  return keff;
}

// GeneralizedIterativeClosestPoint::computeCovariances — registration/include/pcl/registration/impl/gicp.hpp:69-147.
// For every point of `cloud` (the cloud the tree h was built over): k nearest neighbours, covariance of the neighbourhood
// relative to the query (float differences widened to double, :108-111), mean removed (:127-134), SVD, singular values
// replaced by (1, 1, gicp_epsilon) and the matrix reassembled from the columns of U (:136-147).  out: n x 9 doubles,
// row-major.
ORC_API void orc_gicp_covariances(void* h, const float* cloud, size_t n, size_t stride, int k, double gicp_epsilon,
                                  double* out, int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h);
  const int keff = (int)std::min<size_t>((size_t)std::max(k, 0), t.n);
#pragma omp parallel num_threads(nthreads > 0 ? nthreads : 1)
  {
    std::vector<Cand> buf((size_t)std::max(keff, 1));
#pragma omp for schedule(dynamic, 256)
    for (long long i = 0; i < (long long)n; ++i) {
      const float* q = cloud + stride * (size_t)i;
      double* o = out + 9 * (size_t)i;
      for (int e = 0; e < 9; ++e)
        o[e] = 0.0;
      if (!finite3(q) || keff <= 0)
        continue;
      KnnSet rs{buf.data(), keff, 0};
      kd_knn_rec(t, 0, q, rs);
      double mean[3] = {0, 0, 0}, cov[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
      for (int j = 0; j < rs.n; ++j) {
        const float* p = cloud + stride * (size_t)rs.c[j].i;
        const double ptx = p[0] - q[0], pty = p[1] - q[1], ptz = p[2] - q[2];
        mean[0] += ptx; mean[1] += pty; mean[2] += ptz;
        cov[0] += ptx * ptx;
        cov[3] += pty * ptx; cov[4] += pty * pty;
        cov[6] += ptz * ptx; cov[7] += ptz * pty; cov[8] += ptz * ptz;
      }
      const double kk = static_cast<double>(k);
      for (int d = 0; d < 3; ++d)
        mean[d] /= kk;
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c <= r; ++c) {
          cov[3 * r + c] /= kk;
          cov[3 * r + c] -= mean[r] * mean[c];
          cov[3 * c + r] = cov[3 * r + c];
        }
      double U[9], sv[3], V[9];
      svd3<double>(cov, U, sv, V);
      for (int kcol = 0; kcol < 3; ++kcol) {
        const double v = kcol == 2 ? gicp_epsilon : 1.0;
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c)
            o[3 * r + c] += v * U[3 * r + kcol] * U[3 * c + kcol];
      }
    }
  }
}

// brute-force k-NN over the raw cloud (ground truth for the tree itself; same conventions)
ORC_API int orc_knn_bruteforce(const float* pts, size_t n, size_t stride, const float* q, size_t nq,
                               size_t qstride, int k, int32_t* out_idx, float* out_d2)
{
  std::vector<int32_t> valid;
  for (size_t i = 0; i < n; ++i)
    if (finite3(pts + stride * i))
      valid.push_back((int32_t)i);
  int keff = (int)std::min<size_t>((size_t)std::max(k, 0), valid.size());
  if (k <= 0)
    return 0;
  std::vector<Cand> buf((size_t)std::max(keff, 1));
  for (size_t i = 0; i < nq; ++i) {
    KnnSet rs{buf.data(), keff, 0};
    if (keff > 0)
      for (int32_t v : valid)
        rs.offer(Cand{dist2(q + qstride * i, pts + stride * (size_t)v), v});
    for (int j = 0; j < k; ++j) {
      out_idx[i * k + j] = j < rs.n ? rs.c[j].i : -1;
      out_d2[i * k + j] = j < rs.n ? rs.c[j].d : std::numeric_limits<float>::infinity();
    }
  }
  return keff;
}

// ---- radius -----------------------------------------------------------------------------
// KdTreeFLANN::radiusSearch — kdtree_flann.hpp:372-414: r2 = float(radius*radius); max_nn == 0
// or > N => unlimited; otherwise the max_nn nearest inside the ball; ascending by distance
// (sorted_ default true, kdtree/include/pcl/kdtree/kdtree.h:75).
// Two-call protocol: call with out_idx == NULL to get offsets[nq+1], then again with buffers.
ORC_API int orc_radius(void* h, const float* q, size_t nq, size_t qstride, double radius,
                       unsigned max_nn, int64_t* offsets, int32_t* out_idx, float* out_d2,
                       int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h);
  const float r2 = static_cast<float>(radius * radius);
  if (max_nn == 0 || max_nn > t.n)
    max_nn = (unsigned)t.n;
  std::vector<int64_t> counts(nq, 0);
#pragma omp parallel num_threads(nthreads > 0 ? nthreads : 1)
  {
    std::vector<Cand> found;
#pragma omp for schedule(dynamic, 256)
    for (long long i = 0; i < (long long)nq; ++i) {
      found.clear();
      if (t.n)
        kd_radius_rec(t, 0, q + qstride * (size_t)i, r2, found);
      std::sort(found.begin(), found.end(), cand_less);
      size_t m = std::min<size_t>(found.size(), max_nn);
      counts[i] = (int64_t)m;
      if (out_idx) {
        int64_t o = offsets[i];
        for (size_t j = 0; j < m; ++j) {
          out_idx[o + (int64_t)j] = found[j].i;
          out_d2[o + (int64_t)j] = found[j].d;
        }
      }
    }
  }
  if (!out_idx) {
    offsets[0] = 0;
    for (size_t i = 0; i < nq; ++i)
      offsets[i + 1] = offsets[i] + counts[i];
  }
  return 0;
}

// ---- correspondences --------------------------------------------------------------------
// CorrespondenceEstimation::determineCorrespondences —
// registration/include/pcl/registration/impl/correspondence_estimation.hpp:145-218.
// indices == NULL => identity (PCLBase::initCompute, common/include/pcl/impl/pcl_base.hpp:138-171).
ORC_API size_t orc_correspondences(void* h_tgt, const float* src, size_t n_src, size_t sstride,
                                   const int32_t* indices, size_t n_idx, int is_dense,
                                   double max_distance, orc_corr* out, int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h_tgt);
  size_t cnt = indices ? n_idx : n_src;
  const double max_dist_sqr = max_distance * max_distance;
  std::vector<orc_corr> tmp(cnt);
  std::vector<uint8_t> keep(cnt, 0);
  if (t.n == 0)
    return 0;
#pragma omp parallel for schedule(dynamic, 1024) num_threads(nthreads > 0 ? nthreads : 1)
  for (long long i = 0; i < (long long)cnt; ++i) {
    int32_t idx = indices ? indices[i] : (int32_t)i;
    const float* p = src + sstride * (size_t)idx;
    if (!is_dense && !finite3(p))
      continue;
    Cand c;
    KnnSet rs{&c, 1, 0};
    kd_knn_rec(t, 0, p, rs);
    if (c.d > max_dist_sqr)
      continue;
    tmp[i] = orc_corr{idx, c.i, c.d};
    keep[i] = 1;
  }
  size_t m = 0;
  for (size_t i = 0; i < cnt; ++i)
    if (keep[i])
      out[m++] = tmp[i];
  return m;
}

// CorrespondenceEstimation::determineReciprocalCorrespondences — correspondence_estimation.hpp
// :220-311.  h_src is the tree over the (transformed) source cloud; tgt is the raw target cloud.
ORC_API size_t orc_correspondences_reciprocal(void* h_tgt, void* h_src, const float* src,
                                              size_t n_src, size_t sstride, const float* tgt,
                                              size_t tstride, const int32_t* indices, size_t n_idx,
                                              int is_dense, double max_distance, orc_corr* out,
                                              int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h_tgt);
  const KdTree& s = *static_cast<KdTree*>(h_src);
  size_t cnt = indices ? n_idx : n_src;
  const double max_dist_sqr = max_distance * max_distance;
  std::vector<orc_corr> tmp(cnt);
  std::vector<uint8_t> keep(cnt, 0);
  if (t.n == 0 || s.n == 0)
    return 0;
#pragma omp parallel for schedule(dynamic, 1024) num_threads(nthreads > 0 ? nthreads : 1)
  for (long long i = 0; i < (long long)cnt; ++i) {
    int32_t idx = indices ? indices[i] : (int32_t)i;
    const float* p = src + sstride * (size_t)idx;
    if (!is_dense && !finite3(p))
      continue;
    Cand c;
    KnnSet rs{&c, 1, 0};
    kd_knn_rec(t, 0, p, rs);
    if (c.d > max_dist_sqr)
      continue;
    Cand b;
    KnnSet rb{&b, 1, 0};
    kd_knn_rec(s, 0, tgt + tstride * (size_t)c.i, rb);
    if (b.d > max_dist_sqr || idx != b.i)
      continue;
    tmp[i] = orc_corr{idx, c.i, c.d};
    keep[i] = 1;
  }
  size_t m = 0;
  for (size_t i = 0; i < cnt; ++i)
    if (keep[i])
      out[m++] = tmp[i];
  return m;
}

// ---- transformation estimation ----------------------------------------------------------
// T_out: 16 doubles, row-major (a float result is widened exactly).  corr == NULL pairs i<->i.
ORC_API void orc_estimate_svd(const float* src, size_t sstride, const float* tgt, size_t tstride,
                              const orc_corr* corr, size_t n, int scalar_is_double, double* T_out)
{
  std::vector<int32_t> qi, mi;
  if (corr) {
    qi.resize(n);
    mi.resize(n);
    for (size_t i = 0; i < n; ++i) {
      qi[i] = corr[i].index_query;
      mi[i] = corr[i].index_match;
    }
  }
  if (scalar_is_double) {
    double T[16];
    umeyama<double>(src, sstride, tgt, tstride, corr ? qi.data() : nullptr,
                    corr ? mi.data() : nullptr, n, T);
    for (int i = 0; i < 16; ++i)
      T_out[i] = T[i];
  }
  else {
    float T[16];
    umeyama<float>(src, sstride, tgt, tstride, corr ? qi.data() : nullptr,
                   corr ? mi.data() : nullptr, n, T);
    for (int i = 0; i < 16; ++i)
      T_out[i] = T[i];
  }
}

// TransformationEstimationSVD with use_umeyama_ = false — impl/transformation_estimation_svd.hpp:156-225:
// compute3DCentroid (common/impl/centroid.hpp:55-85: sums in Scalar, / n), demeanPointCloud (:933-964),
// getTransformationFromCorrelation: H = src_demean * tgt_demean^T, JacobiSVD, R = V U^T (last column of V negated when
// det(U) det(V) < 0), t = c_tgt - R c_src.
template <typename S>
static void correlation_svd(const float* src, size_t sstride, const float* tgt, size_t tstride, const int32_t* qi,
                            const int32_t* mi, size_t n, S T[16])
{
  S cs[3] = {0, 0, 0}, ct[3] = {0, 0, 0};
  for (size_t i = 0; i < n; ++i) {
    const float* p = src + sstride * (size_t)(qi ? qi[i] : (int32_t)i);
    const float* q = tgt + tstride * (size_t)(mi ? mi[i] : (int32_t)i);
    for (int d = 0; d < 3; ++d) {
      cs[d] += p[d];
      ct[d] += q[d];
    }
  }
  for (int d = 0; d < 3; ++d) {
    cs[d] /= static_cast<S>(n);
    ct[d] /= static_cast<S>(n);
  }
  S H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (size_t i = 0; i < n; ++i) {
    const float* p = src + sstride * (size_t)(qi ? qi[i] : (int32_t)i);
    const float* q = tgt + tstride * (size_t)(mi ? mi[i] : (int32_t)i);
    const S a[3] = {p[0] - cs[0], p[1] - cs[1], p[2] - cs[2]};
    const S b[3] = {q[0] - ct[0], q[1] - ct[1], q[2] - ct[2]};
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        H[3 * r + c] += a[r] * b[c];
  }
  S U[9], sv[3], V[9];
  svd3<S>(H, U, sv, V);
  if (det3<S>(U) * det3<S>(V) < 0)
    for (int x = 0; x < 3; ++x)
      V[3 * x + 2] = -V[3 * x + 2];
  S R[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      S acc = 0;
      for (int k = 0; k < 3; ++k)
        acc += V[3 * r + k] * U[3 * c + k];
      R[3 * r + c] = acc;
    }
  for (int i = 0; i < 16; ++i)
    T[i] = (i % 5 == 0) ? S(1) : S(0);
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c)
      T[4 * r + c] = R[3 * r + c];
    T[4 * r + 3] = ct[r] - (R[3 * r] * cs[0] + R[3 * r + 1] * cs[1] + R[3 * r + 2] * cs[2]);
  }
}

ORC_API void orc_estimate_svd_correlation(const float* src, size_t sstride, const float* tgt, size_t tstride,
                                          const orc_corr* corr, size_t n, int scalar_is_double, double* T_out)
{
  std::vector<int32_t> qi, mi;
  if (corr) {
    qi.resize(n);
    mi.resize(n);
    for (size_t i = 0; i < n; ++i) {
      qi[i] = corr[i].index_query;
      mi[i] = corr[i].index_match;
    }
  }
  if (scalar_is_double) {
    double T[16];
    correlation_svd<double>(src, sstride, tgt, tstride, corr ? qi.data() : nullptr, corr ? mi.data() : nullptr, n, T);
    for (int i = 0; i < 16; ++i)
      T_out[i] = T[i];
  }
  else {
    float T[16];
    correlation_svd<float>(src, sstride, tgt, tstride, corr ? qi.data() : nullptr, corr ? mi.data() : nullptr, n, T);
    for (int i = 0; i < 16; ++i)
      T_out[i] = T[i];
  }
}

ORC_API int orc_estimate_point_to_plane_lls(const float* src, size_t sstride, const float* tgt,
                                            const float* tgt_normals, size_t tstride,
                                            const orc_corr* corr, size_t n, int scalar_is_double,
                                            double* T_out)
{
  std::vector<int32_t> qi, mi;
  if (corr) {
    qi.resize(n);
    mi.resize(n);
    for (size_t i = 0; i < n; ++i) {
      qi[i] = corr[i].index_query;
      mi[i] = corr[i].index_match;
    }
  }
  bool ok;
  if (scalar_is_double) {
    double T[16];
    ok = p2plane_lls<double>(src, sstride, tgt, tgt_normals, tstride, corr ? qi.data() : nullptr,
                             corr ? mi.data() : nullptr, n, T);
    for (int i = 0; i < 16; ++i)
      T_out[i] = T[i];
  }
  else {
    float T[16];
    ok = p2plane_lls<float>(src, sstride, tgt, tgt_normals, tstride, corr ? qi.data() : nullptr,
                            corr ? mi.data() : nullptr, n, T);
    for (int i = 0; i < 16; ++i)
      T_out[i] = T[i];
  }
  return ok ? 0 : -1;
}

ORC_API int orc_estimate_symmetric_lls(const float* src, const float* src_normals, size_t sstride, const float* tgt,
                                       const float* tgt_normals, size_t tstride, const orc_corr* corr, size_t n,
                                       int enforce_same_direction, int scalar_is_double, double* T_out)
{
  std::vector<int32_t> qi, mi;
  if (corr) {
    qi.resize(n);
    mi.resize(n);
    for (size_t i = 0; i < n; ++i) {
      qi[i] = corr[i].index_query;
      mi[i] = corr[i].index_match;
    }
  }
  bool ok;
  if (scalar_is_double) {
    double T[16];
    ok = sym_p2plane_lls<double>(src, src_normals, sstride, tgt, tgt_normals, tstride, corr ? qi.data() : nullptr,
                                 corr ? mi.data() : nullptr, n, enforce_same_direction != 0, T);
    for (int i = 0; i < 16; ++i) T_out[i] = T[i];
  }
  else {
    float T[16];
    ok = sym_p2plane_lls<float>(src, src_normals, sstride, tgt, tgt_normals, tstride, corr ? qi.data() : nullptr,
                                corr ? mi.data() : nullptr, n, enforce_same_direction != 0, T);
    for (int i = 0; i < 16; ++i) T_out[i] = T[i];
  }
  return ok ? 0 : -1;
}

// in-place transform; T row-major 16 doubles (narrowed to float first when !scalar_is_double)
ORC_API void orc_transform(float* pts, size_t n, size_t stride, int normal_off, const double* T,
                           int scalar_is_double, int mode)
{
  if (scalar_is_double)
    transform_points<double>(pts, n, stride, normal_off, T, mode);
  else {
    float Tf[16];
    for (int i = 0; i < 16; ++i)
      Tf[i] = static_cast<float>(T[i]);
    transform_points<float>(pts, n, stride, normal_off, Tf, mode);
  }
}

// ---- correspondence rejectors (SURVEY.md §8f #1) ----------------------------------------------------------
// registration/src/correspondence_rejection_distance.cpp:44-68            keep distance <  max_dist^2 (float), order kept
// registration/src/correspondence_rejection_median_distance.cpp:44-70     keep distance <= median * factor (double), order kept
// registration/src/correspondence_rejection_one_to_one.cpp:44-71          sort by (index_match, distance), first per match
// registration/src/correspondence_rejection_trimmed.cpp:44-63             floor(overlap * n) (>= min) smallest distances
// std::sort in the last two is unstable; canonical tie rule here and on the device: earlier in the input first.
// Distances may be any non-NaN float; -0.0 compares equal to +0.0, and a median that is -0.0 is reported as +0.0.
enum { REJ_DISTANCE = 0, REJ_MEDIAN = 1, REJ_ONE_TO_ONE = 2, REJ_TRIMMED = 3, REJ_SURFACE_NORMAL = 4 };

struct orc_rejector {
  int32_t kind;
  int32_t min_correspondences;  // trimmed: nr_min_correspondences_
  double p;                     // distance: max distance (not squared); median: factor; trimmed: overlap ratio
};

static void apply_rejector(const orc_rejector& r, std::vector<orc_corr>& c, double* median_out)
{
  std::vector<orc_corr> out;
  out.reserve(c.size());
  if (r.kind == REJ_DISTANCE) {
    const float md = static_cast<float>(r.p) * static_cast<float>(r.p);  // setMaximumDistance: max_distance_ = d*d (float)
    for (const auto& x : c)
      if (x.distance < md)
        out.push_back(x);
  }
  else if (r.kind == REJ_MEDIAN) {
    if (c.empty())
      return;
    std::vector<double> d(c.size());
    for (size_t i = 0; i < c.size(); ++i)
      d[i] = c[i].distance;
    std::vector<double> nth(d);
    std::nth_element(nth.begin(), nth.begin() + (nth.size() / 2), nth.end());
    const double med = nth[nth.size() / 2] + 0.0;  // -0.0 -> +0.0
    if (median_out)
      *median_out = med;
    for (size_t i = 0; i < c.size(); ++i)
      if (d[i] <= med * r.p)
        out.push_back(c[i]);
  }
  else if (r.kind == REJ_ONE_TO_ONE) {
    std::vector<orc_corr> in(c);
    std::stable_sort(in.begin(), in.end(), [](const orc_corr& a, const orc_corr& b) {
      return a.index_match < b.index_match || (a.index_match == b.index_match && a.distance < b.distance);
    });
    int32_t last = -1;
    for (const auto& x : in) {
      if (x.index_match < 0)
        continue;
      if (x.index_match != last) {
        out.push_back(x);
        last = x.index_match;
      }
    }
  }
  else {  // trimmed; setOverlapRatio clamps in float (correspondence_rejection_trimmed.h:84), setMinCorrespondences is unsigned
    const float overlap = std::min(1.0f, std::max(0.0f, static_cast<float>(r.p)));
    unsigned keep = static_cast<unsigned>(std::floor(overlap * static_cast<float>(c.size())));
    keep = std::max(keep, static_cast<unsigned>(r.min_correspondences));
    if (keep < c.size()) {
      out = c;
      std::stable_sort(out.begin(), out.end(), [](const orc_corr& a, const orc_corr& b) { return a.distance < b.distance; });
      out.resize(keep);
    }
    else
      return;
  }
  c.swap(out);
}

ORC_API size_t orc_reject(const orc_rejector* r, const orc_corr* in, size_t n, orc_corr* out, double* median_out)
{
  std::vector<orc_corr> c(in, in + n);
  apply_rejector(*r, c, median_out);
  std::copy(c.begin(), c.end(), out);
  return c.size();
}

static inline bool surface_normal_keeps(const float* a, const float* b, double threshold);

// The chain of the ICP loop (icp.hpp:187-201), with one tie rule for every stage: each rejector sees the survivors of
// the one before in source-position order (the order of `c` on entry) and so breaks exact-distance ties by position,
// even after a one-to-one, whose own output is in index_match order; the result is in position order too.  PCL's
// std::sort is unstable, so it defines no other order.  SURFACE_NORMAL reads the normals at sn / tn (stride in floats).
static void apply_chain(const orc_rejector* rej, int n_rej, std::vector<orc_corr>& c, const float* sn, size_t snstride,
                        const float* tn, size_t tnstride, double* median_out)
{
  std::vector<int32_t> query(c.size());
  for (size_t i = 0; i < c.size(); ++i) {  // index_query carries the position while the chain runs
    query[i] = c[i].index_query;
    c[i].index_query = static_cast<int32_t>(i);
  }
  for (int ri = 0; ri < n_rej; ++ri) {
    if (rej[ri].kind == REJ_SURFACE_NORMAL) {
      std::vector<orc_corr> kept;
      for (const auto& x : c)
        if (surface_normal_keeps(sn + snstride * (size_t)query[x.index_query], tn + tnstride * (size_t)x.index_match,
                                 rej[ri].p))
          kept.push_back(x);
      c.swap(kept);
      continue;
    }
    apply_rejector(rej[ri], c, median_out);
    std::sort(c.begin(), c.end(), [](const orc_corr& a, const orc_corr& b) { return a.index_query < b.index_query; });
  }
  for (auto& x : c)
    x.index_query = query[x.index_query];
}

// apply_chain on a list given in position order (kinds DISTANCE to TRIMMED); *median_out: the last MEDIAN stage's median
ORC_API size_t orc_reject_chain(const orc_rejector* rej, int n_rej, const orc_corr* in, size_t n, orc_corr* out,
                                double* median_out)
{
  std::vector<orc_corr> c(in, in + n);
  apply_chain(rej, n_rej, c, nullptr, 0, nullptr, 0, median_out);
  std::copy(c.begin(), c.end(), out);
  return c.size();
}

// ---- correspondence estimators that use normals (SURVEY.md §8f #2) ------------------------
// kind 1: CorrespondenceEstimationNormalShooting::determineCorrespondences —
//   registration/include/pcl/registration/impl/correspondence_estimation_normal_shooting.hpp:66-131: among the k
//   nearest target points pick the one closest to the line through the source point along its normal
//   (|N x V|^2 in double, V = float differences); the gate compares that SQUARED line distance with max_distance
//   itself (:121, kept as in the reference); the stored distance is the squared point distance (:126).
// kind 2: CorrespondenceEstimationBackProjection::determineCorrespondences —
//   impl/correspondence_estimation_backprojection.hpp:66-118: minimise d2 * (2 - cos^2) in float.
// Not covered by the reference (no check there, the query would be UB in FLANN): non-finite source points give no
// correspondence; when every candidate score is NaN the first neighbour is taken (the reference would reuse the
// previous point's min_index).
enum { CORR_NEAREST = 0, CORR_NORMAL_SHOOTING = 1, CORR_BACK_PROJECTION = 2 };

static size_t corr_knn_select(const KdTree& t, int kind, const float* src, size_t n_src, size_t sstride,
                              const float* sn, size_t snstride, const float* tgt, size_t tstride, const float* tn,
                              size_t tnstride, const int32_t* indices, size_t n_idx, int k, double max_distance,
                              orc_corr* out, int nthreads)
{
  size_t cnt = indices ? n_idx : n_src;
  const int keff = (int)std::min<size_t>((size_t)std::max(k, 0), t.n);
  if (keff == 0)
    return 0;
  std::vector<orc_corr> tmp(cnt);
  std::vector<uint8_t> keep(cnt, 0);
#pragma omp parallel num_threads(nthreads > 0 ? nthreads : 1)
  {
    std::vector<Cand> buf((size_t)keff);
#pragma omp for schedule(dynamic, 512)
    for (long long i = 0; i < (long long)cnt; ++i) {
      const int32_t idx = indices ? indices[i] : (int32_t)i;
      const float* p = src + sstride * (size_t)idx;
      if (!finite3(p))
        continue;
      KnnSet rs{buf.data(), keff, 0};
      kd_knn_rec(t, 0, p, rs);
      const float* n = sn + snstride * (size_t)idx;
      int min_j = 0;
      if (kind == CORR_NORMAL_SHOOTING) {
        double min_dist = std::numeric_limits<double>::max();
        const double Nx = n[0], Ny = n[1], Nz = n[2];
        for (int j = 0; j < rs.n; ++j) {
          const float* q = tgt + tstride * (size_t)rs.c[j].i;
          const float vx = q[0] - p[0], vy = q[1] - p[1], vz = q[2] - p[2];
          const double Vx = vx, Vy = vy, Vz = vz;
          const double Cx = Ny * Vz - Nz * Vy, Cy = Nz * Vx - Nx * Vz, Cz = Nx * Vy - Ny * Vx;
          const double dist = (Cx * Cx + Cy * Cy) + Cz * Cz;
          if (dist < min_dist) {
            min_dist = dist;
            min_j = j;
          }
        }
        if (min_dist > max_distance)
          continue;
      }
      else {
        float min_dist = std::numeric_limits<float>::max();
        for (int j = 0; j < rs.n; ++j) {
          const float* m = tn + tnstride * (size_t)rs.c[j].i;
          const float cos_angle = n[0] * m[0] + n[1] * m[1] + n[2] * m[2];
          const float dist = rs.c[j].d * (2.0f - cos_angle * cos_angle);
          if (dist < min_dist) {
            min_dist = dist;
            min_j = j;
          }
        }
        if (min_dist > max_distance)
          continue;
      }
      tmp[i] = orc_corr{idx, rs.c[min_j].i, rs.c[min_j].d};
      keep[i] = 1;
    }
  }
  size_t m = 0;
  for (size_t i = 0; i < cnt; ++i)
    if (keep[i])
      out[m++] = tmp[i];
  return m;
}

ORC_API size_t orc_correspondences_normals(void* h_tgt, int kind, const float* src, size_t n_src, size_t sstride,
                                           const float* sn, size_t snstride, const float* tgt, size_t tstride,
                                           const float* tn, size_t tnstride, const int32_t* indices, size_t n_idx,
                                           int k, double max_distance, orc_corr* out, int nthreads)
{
  return corr_knn_select(*static_cast<KdTree*>(h_tgt), kind, src, n_src, sstride, sn, snstride, tgt, tstride, tn,
                         tnstride, indices, n_idx, k, max_distance, out, nthreads);
}

// CorrespondenceRejectorSurfaceNormal::getRemainingCorrespondences —
// registration/src/correspondence_rejection_surface_normal.cpp:43-66 with the score of
// DataContainer::getCorrespondenceScoreFromNormals (registration/correspondence_rejection.h:378-389): the float dot
// product of the two normals, kept when (double)dot > threshold.
static inline bool surface_normal_keeps(const float* a, const float* b, double threshold)
{
  const float dot = (a[0] * b[0]) + (a[1] * b[1]) + (a[2] * b[2]);
  return static_cast<double>(dot) > threshold;
}

ORC_API size_t orc_reject_surface_normal(const orc_corr* in, size_t n, const float* sn, size_t snstride,
                                         const float* tn, size_t tnstride, double threshold, orc_corr* out)
{
  size_t m = 0;
  for (size_t i = 0; i < n; ++i)
    if (surface_normal_keeps(sn + snstride * (size_t)in[i].index_query, tn + tnstride * (size_t)in[i].index_match,
                             threshold))
      out[m++] = in[i];
  return m;
}

// ---- ICP --------------------------------------------------------------------------------
struct orc_icp_params {
  int32_t max_iterations;            // registration.h:566 default 10
  int32_t use_reciprocal;            // icp.h setUseReciprocalCorrespondences
  int32_t estimator;                 // 0 = SVD (Umeyama), 1 = point-to-plane LLS
  int32_t scalar_is_double;          // Scalar template argument
  int32_t with_normals_transform;    // 0: IterativeClosestPoint::transformCloud, 1: ...WithNormals
  int32_t source_has_normals;        // rotate source normals (float offset 4) while transforming
  int32_t is_dense;                  // input_->is_dense
  int32_t nthreads;
  double max_correspondence_distance;        // registration.h:117 default sqrt(DBL_MAX)
  double transformation_epsilon;             // registration.h:588 default 0
  double transformation_rotation_epsilon;    // default 0 (= unused)
  double euclidean_fitness_epsilon;          // registration.h:116 default -DBL_MAX
  int32_t correspondence_kind;               // 0 nearest, 1 normal shooting, 2 back projection (need source normals)
  int32_t correspondence_k;                  // k_ of the two normal-based estimators (default 10)
};

struct orc_icp_result {
  double final_transformation[16];   // row-major
  double last_transformation[16];
  int32_t converged;
  int32_t state;
  int32_t iterations;
  int32_t n_correspondences;         // of the last evaluated iteration
  double mse;                        // of the last evaluated iteration
  long long total_correspondences;   // summed over the iterations (throughput accounting in bench.py)
};

// The knobs of the loop that sit outside Registration's own setters: DefaultConvergenceCriteria's members
// (default_convergence_criteria.h:148-152, 307-310), TransformationEstimationSVD(use_umeyama = false)
// (transformation_estimation_svd.h:69) and setEnforceSameDirectionNormals (icp.h:402-418).  nullptr = the defaults.
struct orc_icp_ext {
  int32_t failure_after_max_iter;             // default 0
  int32_t max_iterations_similar_transforms;  // default 0
  int32_t svd_no_umeyama;                     // default 0
  int32_t enforce_same_direction_normals;     // default 1
  double mse_threshold_absolute;              // default 1e-12
};

template <typename S>
static void icp_run(const orc_icp_params& P, const float* src, size_t n_s, size_t ss,
                    const int32_t* indices, size_t n_idx, const float* tgt, size_t n_t, size_t ts,
                    const double* guess, orc_icp_result& R, float* out_cloud, void* prebuilt_tree = nullptr,
                    const orc_rejector* rejectors = nullptr, int n_rejectors = 0, const orc_icp_ext* X = nullptr,
                    orc_corr* last_corr = nullptr, size_t* n_last_corr = nullptr, double* prev_mse = nullptr)
{
  // Registration::align (registration/.../impl/registration.hpp:172-221) +
  // IterativeClosestPoint::computeTransformation (impl/icp.hpp:113-268)
  const int noff = P.source_has_normals ? 4 : -1;
  const int tmode = P.with_normals_transform ? 1 : 0;
  // Registration::initCompute rebuilds the target tree only when the target changed
  // (registration.hpp:84-87): a caller that keeps the target passes the tree it already has.
  KdTree* tree = prebuilt_tree ? static_cast<KdTree*>(prebuilt_tree)
                               : static_cast<KdTree*>(orc_index_build(tgt, n_t, ts, nullptr, 0));
  S final_T[16], T[16], G[16];
  bool guess_is_identity = true;
  for (int i = 0; i < 16; ++i) {
    G[i] = static_cast<S>(guess ? guess[i] : ((i % 5 == 0) ? 1.0 : 0.0));
    if (G[i] != ((i % 5 == 0) ? S(1) : S(0)))
      guess_is_identity = false;
    final_T[i] = G[i];
    T[i] = (i % 5 == 0) ? S(1) : S(0);
  }
  std::vector<float> cur(src, src + n_s * ss);  // input_transformed
  if (!guess_is_identity)
    transform_points<S>(cur.data(), n_s, ss, noff, G, tmode);
  Convergence<S> conv;
  conv.max_iterations = P.max_iterations;
  conv.mse_threshold_relative = P.euclidean_fitness_epsilon;
  conv.translation_threshold = P.transformation_epsilon;
  if (P.transformation_rotation_epsilon > 0)
    conv.rotation_threshold = P.transformation_rotation_epsilon;
  if (X) {
    conv.failure_after_max_iter = X->failure_after_max_iter != 0;
    conv.max_iterations_similar_transforms = X->max_iterations_similar_transforms;
    conv.mse_threshold_absolute = X->mse_threshold_absolute;
  }
  if (prev_mse)
    conv.prev_mse = *prev_mse;
  std::vector<orc_corr> corr(indices ? n_idx : n_s);
  int iterations = 0;
  bool converged = false;
  size_t nc = 0;
  double mse = 0;
  long long total_nc = 0;
  do {
    if (P.use_reciprocal) {
      KdTree* stree = static_cast<KdTree*>(orc_index_build(cur.data(), n_s, ss, indices, indices ? n_idx : 0));
      nc = orc_correspondences_reciprocal(tree, stree, cur.data(), n_s, ss, tgt, ts, indices, n_idx,
                                          P.is_dense, P.max_correspondence_distance, corr.data(),
                                          P.nthreads);
      orc_index_free(stree);
    }
    else if (P.correspondence_kind != CORR_NEAREST)
      // icp.hpp:166-180: the estimator sees the transformed source and its rotated normals
      nc = corr_knn_select(*tree, P.correspondence_kind, cur.data(), n_s, ss, cur.data() + 4, ss, tgt, ts, tgt + 4, ts,
                           indices, n_idx, P.correspondence_k, P.max_correspondence_distance, corr.data(), P.nthreads);
    else
      nc = orc_correspondences(tree, cur.data(), n_s, ss, indices, n_idx, P.is_dense,
                               P.max_correspondence_distance, corr.data(), P.nthreads);
    if (n_rejectors > 0) {  // icp.hpp:187-201: each rejector filters the previous one's survivors (in position order)
      std::vector<orc_corr> cc(corr.begin(), corr.begin() + nc);
      // surface normal: the normals of the transformed source vs the target's
      apply_chain(rejectors, n_rejectors, cc, cur.data() + 4, ss, tgt + 4, ts, nullptr);
      nc = cc.size();
      std::copy(cc.begin(), cc.end(), corr.begin());
    }
    total_nc += (long long)nc;
    if (nc < 3) {  // min_number_correspondences_, registration.h:621; icp.hpp:204-213
      conv.state = NO_CORRESPONDENCES;
      converged = false;
      break;
    }
    std::vector<int32_t> qi(nc), mi(nc);
    mse = 0;
    for (size_t i = 0; i < nc; ++i) {
      qi[i] = corr[i].index_query;
      mi[i] = corr[i].index_match;
      mse += corr[i].distance;
    }
    mse /= static_cast<double>(nc);
    if (P.estimator == 0 && X && X->svd_no_umeyama)
      correlation_svd<S>(cur.data(), ss, tgt, ts, qi.data(), mi.data(), nc, T);
    else if (P.estimator == 0)
      umeyama<S>(cur.data(), ss, tgt, ts, qi.data(), mi.data(), nc, T);
    else if (P.estimator == 1)
      p2plane_lls<S>(cur.data(), ss, tgt, tgt + 4, ts, qi.data(), mi.data(), nc, T);
    else  // symmetric objective; setEnforceSameDirectionNormals(true) is the class default (icp.h:366-371)
      sym_p2plane_lls<S>(cur.data(), cur.data() + 4, ss, tgt, tgt + 4, ts, qi.data(), mi.data(), nc,
                         X ? X->enforce_same_direction_normals != 0 : true, T);
    transform_points<S>(cur.data(), n_s, ss, noff, T, tmode);
    mat4_mul<S>(T, final_T, final_T);
    ++iterations;
    converged = conv.has_converged(iterations, T, mse);
  } while (conv.state == NOT_CONVERGED);
  for (int i = 0; i < 16; ++i) {
    R.final_transformation[i] = final_T[i];
    R.last_transformation[i] = T[i];
  }
  if (prev_mse)
    *prev_mse = conv.prev_mse;
  R.converged = converged ? 1 : 0;
  R.state = conv.state;
  R.iterations = iterations;
  R.n_correspondences = (int32_t)nc;
  R.mse = mse;
  R.total_correspondences = total_nc;
  if (last_corr) {  // Registration::correspondences_ after the loop: those of the last evaluated iteration
    std::copy(corr.begin(), corr.begin() + nc, last_corr);
    *n_last_corr = nc;
  }
  if (out_cloud) {  // output = *input_; transformCloud(*input_, output, final) — icp.hpp:265-267
    std::memcpy(out_cloud, src, n_s * ss * sizeof(float));
    transform_points<S>(out_cloud, n_s, ss, noff, final_T, tmode);
  }
  if (!prebuilt_tree)
    orc_index_free(tree);
}

ORC_API void orc_icp_align(const orc_icp_params* P, const float* src, size_t n_s, size_t sstride,
                           const int32_t* indices, size_t n_idx, const float* tgt, size_t n_t,
                           size_t tstride, const double* guess, orc_icp_result* R, float* out_cloud)
{
  if (P->scalar_is_double)
    icp_run<double>(*P, src, n_s, sstride, indices, n_idx, tgt, n_t, tstride, guess, *R, out_cloud);
  else
    icp_run<float>(*P, src, n_s, sstride, indices, n_idx, tgt, n_t, tstride, guess, *R, out_cloud);
}

ORC_API void orc_icp_align_tree(const orc_icp_params* P, void* h_tgt, const float* src, size_t n_s,
                                size_t sstride, const int32_t* indices, size_t n_idx, const float* tgt,
                                size_t n_t, size_t tstride, const double* guess, orc_icp_result* R,
                                float* out_cloud)
{
  if (P->scalar_is_double)
    icp_run<double>(*P, src, n_s, sstride, indices, n_idx, tgt, n_t, tstride, guess, *R, out_cloud, h_tgt);
  else
    icp_run<float>(*P, src, n_s, sstride, indices, n_idx, tgt, n_t, tstride, guess, *R, out_cloud, h_tgt);
}

// Everything at once: rejector chain + kept target tree + source indices + guess + the criteria / estimator knobs, and
// the correspondences of the last evaluated iteration (capacity: the number of indexed source points).
ORC_API void orc_icp_align_full(const orc_icp_params* P, const orc_icp_ext* X, const orc_rejector* rej, int n_rej,
                                void* h_tgt, const float* src, size_t n_s, size_t sstride, const int32_t* indices,
                                size_t n_idx, const float* tgt, size_t n_t, size_t tstride, const double* guess,
                                orc_icp_result* R, float* out_cloud, orc_corr* last_corr, size_t* n_last_corr)
{
  if (P->scalar_is_double)
    icp_run<double>(*P, src, n_s, sstride, indices, n_idx, tgt, n_t, tstride, guess, *R, out_cloud, h_tgt, rej, n_rej, X,
                    last_corr, n_last_corr);
  else
    icp_run<float>(*P, src, n_s, sstride, indices, n_idx, tgt, n_t, tstride, guess, *R, out_cloud, h_tgt, rej, n_rej, X,
                   last_corr, n_last_corr);
}

// orc_icp_align_full on a criteria object that outlives one align (icp.h:155): *prev_mse is its
// correspondences_prev_mse_ (default_convergence_criteria.h:283) when the align starts, and is where the align leaves it.
ORC_API void orc_icp_align_carry(const orc_icp_params* P, const orc_icp_ext* X, const orc_rejector* rej, int n_rej,
                                 void* h_tgt, const float* src, size_t n_s, size_t sstride, const int32_t* indices,
                                 size_t n_idx, const float* tgt, size_t n_t, size_t tstride, const double* guess,
                                 orc_icp_result* R, float* out_cloud, orc_corr* last_corr, size_t* n_last_corr,
                                 double* prev_mse)
{
  if (P->scalar_is_double)
    icp_run<double>(*P, src, n_s, sstride, indices, n_idx, tgt, n_t, tstride, guess, *R, out_cloud, h_tgt, rej, n_rej, X,
                    last_corr, n_last_corr, prev_mse);
  else
    icp_run<float>(*P, src, n_s, sstride, indices, n_idx, tgt, n_t, tstride, guess, *R, out_cloud, h_tgt, rej, n_rej, X,
                   last_corr, n_last_corr, prev_mse);
}

// Registration::getFitnessScore — registration/.../impl/registration.hpp:134-168
ORC_API double orc_fitness_score(void* h_tgt, const float* src, size_t n_s, size_t sstride,
                                 const int32_t* indices, size_t n_idx, int is_dense,
                                 const double* final_T, int scalar_is_double, double max_range,
                                 int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h_tgt);
  size_t cnt = (indices && n_idx != n_s) ? n_idx : n_s;
  std::vector<float> pts(cnt * 4);
  for (size_t i = 0; i < cnt; ++i) {
    const float* p = src + sstride * (size_t)((indices && n_idx != n_s) ? indices[i] : (int32_t)i);
    pts[4 * i] = p[0];
    pts[4 * i + 1] = p[1];
    pts[4 * i + 2] = p[2];
    pts[4 * i + 3] = 1.0f;
  }
  orc_transform(pts.data(), cnt, 4, -1, final_T, scalar_is_double, 1);
  double score = 0;
  long long nr = 0;
  (void)nthreads;
  for (size_t i = 0; i < cnt; ++i) {
    if (!is_dense && !finite3(&pts[4 * i]))
      continue;
    Cand c;
    KnnSet rs{&c, 1, 0};
    kd_knn_rec(t, 0, &pts[4 * i], rs);
    if (c.d <= max_range) {
      score += c.d;
      ++nr;
    }
  }
  return nr > 0 ? score / (double)nr : std::numeric_limits<double>::max();
}

// ---- VoxelGrid --------------------------------------------------------------------------
// VoxelGrid<PointT>::applyFilter — filters/include/pcl/filters/impl/voxel_grid.hpp:596-814
// (no filter field), getMinMax3D common/include/pcl/common/impl/common.hpp:348, centroid =
// AccumulatorXYZ (common/include/pcl/common/impl/accumulators.hpp:68-85): float sums, / n.
// out: capacity n*4 floats (x,y,z,1).  Returns the number of output points, or -1 when the
// INT32 overflow guard trips (reference then copies the input unfiltered, :620-629).
// normal_off >= 0 (float offset of normal_x inside a record) additionally averages the normal and the curvature like
// CentroidPoint does under downsample_all_data_ (voxel_grid.hpp:796-806; AccumulatorNormal / AccumulatorCurvature,
// accumulators.hpp:86-133): out_nc gets 8 floats per voxel {normalised 4-vector sum, mean curvature, 0, 0, 0}.
static long long voxelgrid_impl(const float* pts, size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                                int is_dense, const float leaf[3], unsigned min_pts, float* out, long normal_off,
                                float* out_nc)
{
  size_t cnt = indices ? n_idx : n;
  float inv[3] = {1.0f / leaf[0], 1.0f / leaf[1], 1.0f / leaf[2]};
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (size_t i = 0; i < cnt; ++i) {
    const float* p = pts + stride * (size_t)(indices ? indices[i] : (int32_t)i);
    if (!is_dense && !finite3(p))
      continue;
    for (int d = 0; d < 3; ++d) {
      mn[d] = std::min(mn[d], p[d]);
      mx[d] = std::max(mx[d], p[d]);
    }
  }
  int64_t dx = static_cast<int64_t>((mx[0] - mn[0]) * inv[0]) + 1;
  int64_t dy = static_cast<int64_t>((mx[1] - mn[1]) * inv[1]) + 1;
  int64_t dz = static_cast<int64_t>((mx[2] - mn[2]) * inv[2]) + 1;
  if (dx * dy * dz > static_cast<int64_t>(std::numeric_limits<int32_t>::max()))
    return -1;
  int min_b[3], max_b[3], div_b[3];
  for (int d = 0; d < 3; ++d) {
    min_b[d] = static_cast<int>(std::floor(mn[d] * inv[d]));
    max_b[d] = static_cast<int>(std::floor(mx[d] * inv[d]));
    div_b[d] = max_b[d] - min_b[d] + 1;
  }
  int mul[3] = {1, div_b[0], div_b[0] * div_b[1]};
  std::vector<std::pair<unsigned, int32_t>> iv;
  iv.reserve(cnt);
  for (size_t i = 0; i < cnt; ++i) {
    int32_t ci = indices ? indices[i] : (int32_t)i;
    const float* p = pts + stride * (size_t)ci;
    if (!is_dense && !finite3(p))
      continue;
    int ijk0 = static_cast<int>(std::floor(p[0] * inv[0]) - static_cast<float>(min_b[0]));
    int ijk1 = static_cast<int>(std::floor(p[1] * inv[1]) - static_cast<float>(min_b[1]));
    int ijk2 = static_cast<int>(std::floor(p[2] * inv[2]) - static_cast<float>(min_b[2]));
    int idx = ijk0 * mul[0] + ijk1 * mul[1] + ijk2 * mul[2];
    iv.emplace_back(static_cast<unsigned>(idx), ci);
  }
  std::stable_sort(iv.begin(), iv.end(),
                   [](const std::pair<unsigned, int32_t>& a, const std::pair<unsigned, int32_t>& b) {
                     return a.first < b.first;
                   });
  long long total = 0;
  size_t index = 0;
  while (index < iv.size()) {
    size_t i = index + 1;
    while (i < iv.size() && iv[i].first == iv[index].first)
      ++i;
    if (i - index >= min_pts) {
      float c[3] = {0, 0, 0};
      for (size_t li = index; li < i; ++li) {
        const float* p = pts + stride * (size_t)iv[li].second;
        c[0] += p[0];
        c[1] += p[1];
        c[2] += p[2];
      }
      float fn = static_cast<float>(i - index);
      out[4 * total + 0] = c[0] / fn;
      out[4 * total + 1] = c[1] / fn;
      out[4 * total + 2] = c[2] / fn;
      out[4 * total + 3] = 1.0f;
      if (normal_off >= 0 && out_nc) {
        float nv[4] = {0, 0, 0, 0}, cv = 0;
        for (size_t li = index; li < i; ++li) {
          const float* p = pts + stride * (size_t)iv[li].second + normal_off;
          nv[0] += p[0]; nv[1] += p[1]; nv[2] += p[2]; nv[3] += p[3];
          cv += p[4];
        }
        const float sq = (nv[0] * nv[0] + nv[1] * nv[1]) + (nv[2] * nv[2] + nv[3] * nv[3]);
        if (sq > 0.f) {
          const float nrm = std::sqrt(sq);
          for (int d = 0; d < 4; ++d) nv[d] /= nrm;
        }
        float* o = out_nc + 8 * total;
        o[0] = nv[0]; o[1] = nv[1]; o[2] = nv[2]; o[3] = nv[3];
        o[4] = cv / fn; o[5] = o[6] = o[7] = 0.f;
      }
      ++total;
    }
    index = i;
  }
  return total;
}

ORC_API long long orc_voxelgrid(const float* pts, size_t n, size_t stride, const int32_t* indices,
                                size_t n_idx, int is_dense, const float leaf[3], unsigned min_pts,
                                float* out)
{
  return voxelgrid_impl(pts, n, stride, indices, n_idx, is_dense, leaf, min_pts, out, -1, nullptr);
}

ORC_API long long orc_voxelgrid_normals(const float* pts, size_t n, size_t stride, const int32_t* indices,
                                        size_t n_idx, int is_dense, const float leaf[3], unsigned min_pts,
                                        float* out, long normal_off, float* out_nc)
{
  return voxelgrid_impl(pts, n, stride, indices, n_idx, is_dense, leaf, min_pts, out, normal_off, out_nc);
}

// ---- normals ----------------------------------------------------------------------------
// computePointNormal over an explicit neighbour list (test_normal_estimation.cpp:106-127 shape)
ORC_API int orc_point_normal(const float* cloud, size_t stride, int is_dense, const int32_t* idx,
                             size_t k, float out[4])
{
  return point_normal(cloud, stride, is_dense != 0, idx, k, out) ? 1 : 0;
}

// NormalEstimation::computeFeature with k-NN — features/include/pcl/features/impl/normal_3d.hpp
// :47-96; neighbours come from the index built over `surface` (== cloud here), query points are
// cloud[indices].  out: cnt*4 floats (nx,ny,nz,curvature).  Returns 1 if all outputs are finite
// (output.is_dense).
ORC_API int orc_normals_knn(void* h, const float* cloud, size_t n, size_t stride,
                            const int32_t* indices, size_t n_idx, int is_dense, int k,
                            const float vp[3], float* out, int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h);
  size_t cnt = indices ? n_idx : n;
  int keff = (int)std::min<size_t>((size_t)std::max(k, 0), t.n);
  int dense_out = 1;
  const float qnan = std::numeric_limits<float>::quiet_NaN();
#pragma omp parallel num_threads(nthreads > 0 ? nthreads : 1)
  {
    std::vector<Cand> buf((size_t)std::max(keff, 1));
    std::vector<int32_t> nn((size_t)std::max(keff, 1));
#pragma omp for schedule(dynamic, 512)
    for (long long i = 0; i < (long long)cnt; ++i) {
      const float* p = cloud + stride * (size_t)(indices ? indices[i] : (int32_t)i);
      float* o = out + 4 * (size_t)i;
      bool ok = keff > 0 && (is_dense || finite3(p));
      if (ok) {
        KnnSet rs{buf.data(), keff, 0};
        kd_knn_rec(t, 0, p, rs);
        for (int j = 0; j < rs.n; ++j)
          nn[j] = rs.c[j].i;
        ok = point_normal(cloud, stride, is_dense != 0, nn.data(), (size_t)rs.n, o);
      }
      if (!ok) {
        o[0] = o[1] = o[2] = o[3] = qnan;
#pragma omp atomic write
        dense_out = 0;
        continue;
      }
      flip_to_viewpoint(p, vp, o);
    }
  }
  return dense_out;
}

// NormalEstimation with setRadiusSearch — Feature::initCompute picks radiusSearch(point, radius) with max_nn = 0
// (features/include/pcl/features/impl/feature.hpp:149-166), so the neighbourhood is every point with d2 < r2 in
// ascending (d2, index) order; the rest is identical to the k-NN path (normal_3d.hpp:47-96).
ORC_API int orc_normals_radius(void* h, const float* cloud, size_t n, size_t stride, const int32_t* indices,
                               size_t n_idx, int is_dense, double radius, const float vp[3], float* out, int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h);
  size_t cnt = indices ? n_idx : n;
  const float r2 = static_cast<float>(radius * radius);
  int dense_out = 1;
  const float qnan = std::numeric_limits<float>::quiet_NaN();
#pragma omp parallel num_threads(nthreads > 0 ? nthreads : 1)
  {
    std::vector<Cand> found;
    std::vector<int32_t> nn;
#pragma omp for schedule(dynamic, 512)
    for (long long i = 0; i < (long long)cnt; ++i) {
      const float* p = cloud + stride * (size_t)(indices ? indices[i] : (int32_t)i);
      float* o = out + 4 * (size_t)i;
      bool ok = t.n > 0 && (is_dense || finite3(p));
      if (ok) {
        found.clear();
        kd_radius_rec(t, 0, p, r2, found);
        std::sort(found.begin(), found.end(), cand_less);
        nn.resize(found.size());
        for (size_t j = 0; j < found.size(); ++j)
          nn[j] = found[j].i;
        ok = point_normal(cloud, stride, is_dense != 0, nn.data(), nn.size(), o);
      }
      if (!ok) {
        o[0] = o[1] = o[2] = o[3] = qnan;
#pragma omp atomic write
        dense_out = 0;
        continue;
      }
      flip_to_viewpoint(p, vp, o);
    }
  }
  return dense_out;
}

// ---- Euclidean clustering (SURVEY.md §8f #4) ---------------------------------------------------------------------
// pcl::extractEuclideanClusters, indices form — segmentation/include/pcl/segmentation/impl/extract_clusters.hpp
// :124-223: breadth-first flood fill, one radiusSearch(point, tolerance) per queue entry, over the points the tree
// holds; the tolerance reaches it as float (:246).  out_labels[i] = smallest index of point i's cluster (the seed, since
// seeds are taken in ascending order and a cluster's indices are sorted at :208), -1 for points the tree does not hold.
// Size window and ordering by size (:196, :249) are applied by the caller on the labels.
ORC_API void orc_cluster_labels(void* h, size_t n_cloud, double tolerance, int32_t* out_labels)
{
  const KdTree& t = *static_cast<KdTree*>(h);
  std::fill(out_labels, out_labels + n_cloud, -1);
  const double tol = static_cast<double>(static_cast<float>(tolerance));
  const float r2 = static_cast<float>(tol * tol);
  // tree slot of every original index it holds, so a queue entry's coordinates can be looked up
  std::vector<int32_t> slot_of(n_cloud, -1);
  for (size_t i = 0; i < t.n; ++i)
    slot_of[(size_t)t.orig[i]] = (int32_t)i;
  std::vector<Cand> found;
  std::vector<int32_t> queue;
  for (size_t seed = 0; seed < n_cloud; ++seed) {
    if (slot_of[seed] < 0 || out_labels[seed] >= 0)
      continue;
    queue.clear();
    queue.push_back((int32_t)seed);
    out_labels[seed] = (int32_t)seed;
    for (size_t qi = 0; qi < queue.size(); ++qi) {
      found.clear();
      kd_radius_rec(t, 0, &t.pts[3 * (size_t)slot_of[(size_t)queue[qi]]], r2, found);
      for (const Cand& c : found)
        if (out_labels[(size_t)c.i] < 0) {
          out_labels[(size_t)c.i] = (int32_t)seed;
          queue.push_back(c.i);
        }
    }
  }
}

// ---- k-NN statistics + the two outlier filters built on them (SURVEY.md §8f #4) ---------------------------
// out_mean[i] = float( sum_{j=1..k'-1} sqrt(double(d2_j)) / (k'-1) ), k' = min(k, #indexed points), j = 0 is the query
//               itself (filters/include/pcl/filters/impl/statistical_outlier_removal.hpp:88-97); 0 for non-finite queries
// out_kth[i]  = d2 of the k-th neighbour (index k-1), +inf when fewer than k points are indexed
ORC_API void orc_knn_stats(void* h, const float* cloud, size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                           int k, float* out_mean, float* out_kth, int nthreads)
{
  const KdTree& t = *static_cast<KdTree*>(h);
  size_t cnt = indices ? n_idx : n;
  int keff = (int)std::min<size_t>((size_t)std::max(k, 0), t.n);
#pragma omp parallel num_threads(nthreads > 0 ? nthreads : 1)
  {
    std::vector<Cand> buf((size_t)std::max(keff, 1));
#pragma omp for schedule(dynamic, 512)
    for (long long i = 0; i < (long long)cnt; ++i) {
      const float* p = cloud + stride * (size_t)(indices ? indices[i] : (int32_t)i);
      float mean = 0.0f, kth = std::numeric_limits<float>::infinity();
      if (finite3(p) && keff > 0) {
        KnnSet rs{buf.data(), keff, 0};
        kd_knn_rec(t, 0, p, rs);
        double sum = 0.0;
        for (int j = 1; j < rs.n; ++j)
          sum += std::sqrt(static_cast<double>(rs.c[j].d));
        if (rs.n > 1)
          mean = static_cast<float>(sum / (rs.n - 1));
        if (rs.n == k)
          kth = rs.c[k - 1].d;
      }
      if (out_mean) out_mean[i] = mean;
      if (out_kth) out_kth[i] = kth;
    }
  }
}

// StatisticalOutlierRemoval::applyFilterIndices — statistical_outlier_removal.hpp:47-135.  keep[i] in {0,1}.
ORC_API size_t orc_sor(void* h, const float* cloud, size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                       int mean_k, double std_mul, int negative, uint8_t* keep, int nthreads)
{
  size_t cnt = indices ? n_idx : n;
  std::vector<float> dist(cnt);
  orc_knn_stats(h, cloud, n, stride, indices, n_idx, mean_k + 1, dist.data(), nullptr, nthreads);
  long long valid = 0;
  for (size_t i = 0; i < cnt; ++i)
    if (finite3(cloud + stride * (size_t)(indices ? indices[i] : (int32_t)i)))
      ++valid;
  double sum = 0, sq_sum = 0;
  for (float d : dist) {
    sum += d;
    sq_sum += d * d;
  }
  double mean = sum / static_cast<double>(valid);
  double variance = (sq_sum - sum * sum / static_cast<double>(valid)) / (static_cast<double>(valid) - 1);
  double thr = mean + std_mul * std::sqrt(variance);
  size_t kept = 0;
  for (size_t i = 0; i < cnt; ++i) {
    bool removed = (!negative && dist[i] > thr) || (negative && dist[i] <= thr);
    keep[i] = removed ? 0 : 1;
    kept += keep[i];
  }
  return kept;
}

// RadiusOutlierRemoval::applyFilterIndices — radius_outlier_removal.hpp:49-179 (dense: k-NN rule with <=; non-dense:
// radius rule with the strict FLANN comparison).
ORC_API size_t orc_ror(void* h, const float* cloud, size_t n, size_t stride, const int32_t* indices, size_t n_idx,
                       int is_dense, double radius, int min_pts, int negative, uint8_t* keep, int nthreads)
{
  size_t cnt = indices ? n_idx : n;
  const int mean_k = min_pts + 1;
  std::vector<float> kth(cnt);
  orc_knn_stats(h, cloud, n, stride, indices, n_idx, mean_k, nullptr, kth.data(), nthreads);
  const double nn_dists_max = radius * radius;
  const float r2f = static_cast<float>(radius * radius);
  size_t kept = 0;
  for (size_t i = 0; i < cnt; ++i) {
    const float* p = cloud + stride * (size_t)(indices ? indices[i] : (int32_t)i);
    bool k = true;
    if (is_dense) {
      if (std::isfinite(kth[i])) {  // k == mean_k neighbours found
        if ((!negative && nn_dists_max < kth[i]) || (negative && nn_dists_max >= kth[i]))
          k = false;
      }
      else if (!negative)
        k = false;
    }
    else {
      if (!finite3(p))
        k = false;
      else {
        const bool enough = kth[i] < r2f;  // radiusSearch found min_pts + 1 neighbours (strict d2 < r2)
        if ((!negative && !enough) || (negative && enough))
          k = false;
      }
    }
    keep[i] = k ? 1 : 0;
    kept += keep[i];
  }
  return kept;
}

ORC_API int orc_max_threads()
{
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
