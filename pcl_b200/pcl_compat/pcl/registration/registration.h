// pcl/registration/registration.h + icp.h — pcl::Registration / pcl::IterativeClosestPoint[WithNormals] whose
// computeTransformation runs the device-resident loop of libpclb200 (pclb200_icp_* session).
// Reference: registration/include/pcl/registration/registration.h:56-700, impl/registration.hpp:45-221,
// icp.h:97-456, impl/icp.hpp:113-318, default_convergence_criteria.h:64-326.
#pragma once
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <functional>
#include <type_traits>
#include <limits>
#include <memory>
#include <string>

#include "../search/kdtree.h"
#include <algorithm>
#include <vector>

#include "correspondence_estimation.h"
#include "../conversions.h"
#include "correspondence_rejection.h"
#include "transformation_estimation.h"

namespace pcl {
namespace registration {
// default_convergence_criteria.h:75-83 — the state enum and the accessor PCL users reach through getConvergeCriteria()
template <typename Scalar = float>
class DefaultConvergenceCriteria {
public:
  using Ptr = std::shared_ptr<DefaultConvergenceCriteria<Scalar>>;
  enum ConvergenceState {
    CONVERGENCE_CRITERIA_NOT_CONVERGED = PCLB200_CONV_NOT_CONVERGED,
    CONVERGENCE_CRITERIA_ITERATIONS = PCLB200_CONV_ITERATIONS,
    CONVERGENCE_CRITERIA_TRANSFORM = PCLB200_CONV_TRANSFORM,
    CONVERGENCE_CRITERIA_ABS_MSE = PCLB200_CONV_ABS_MSE,
    CONVERGENCE_CRITERIA_REL_MSE = PCLB200_CONV_REL_MSE,
    CONVERGENCE_CRITERIA_NO_CORRESPONDENCES = PCLB200_CONV_NO_CORRESPONDENCES,
    CONVERGENCE_CRITERIA_FAILURE_AFTER_MAX_ITERATIONS = PCLB200_CONV_FAILURE_AFTER_MAX_ITERATIONS
  };
  ConvergenceState getConvergenceState() const { return state_; }
  void setFailureAfterMaximumIterations(bool f) { failure_after_max_iter_ = f; }
  bool getFailureAfterMaximumIterations() const { return failure_after_max_iter_; }
  void setMaximumIterationsSimilarTransforms(int n) { max_iterations_similar_transforms_ = n; }
  int getMaximumIterationsSimilarTransforms() const { return max_iterations_similar_transforms_; }
  void setAbsoluteMSE(double v) { mse_threshold_absolute_ = v; }
  double getAbsoluteMSE() const { return mse_threshold_absolute_; }
  // default_convergence_criteria.h:130-205.  As in the reference, align() overwrites the maximum iterations, the
  // relative MSE and the translation threshold with Registration's own setters' values (icp.hpp:157-161), and the
  // rotation threshold only when setTransformationRotationEpsilon(> 0) was called: a threshold set HERE is what an
  // align() without that call uses.
  void setMaximumIterations(int n) { max_iterations_ = n; }
  int getMaximumIterations() const { return max_iterations_; }
  void setRotationThreshold(double cos_angle) { rotation_threshold_ = cos_angle; }
  double getRotationThreshold() const { return rotation_threshold_; }
  void setTranslationThreshold(double squared) { translation_threshold_ = squared; }
  double getTranslationThreshold() const { return translation_threshold_; }
  void setRelativeMSE(double v) { mse_threshold_relative_ = v; }
  double getRelativeMSE() const { return mse_threshold_relative_; }
  // written by Registration after every run
  ConvergenceState state_ = CONVERGENCE_CRITERIA_NOT_CONVERGED;
  bool failure_after_max_iter_ = false;
  int max_iterations_similar_transforms_ = 0;
  double mse_threshold_absolute_ = 1e-12;
  int max_iterations_ = 100;                // default_convergence_criteria.h:104-113
  double rotation_threshold_ = 0.99999;
  double translation_threshold_ = 3e-4 * 3e-4;
  double mse_threshold_relative_ = 0.00001;
  // correspondences_prev_mse_ (default_convergence_criteria.h:283): written only when no criterion fired, never reset,
  // so it carries from one align() of the owning object to the next.  The staged loop keeps it here; the device loop
  // keeps its own in the pclb200_icp session, which carries it the same way.
  double prev_mse_ = std::numeric_limits<double>::max();
};
}  // namespace registration

template <typename PointSource, typename PointTarget, typename Scalar = float>
class Registration : public PCLBase<PointSource> {
public:
  using Matrix4 = Eigen::Matrix<Scalar, 4, 4>;
  using Ptr = std::shared_ptr<Registration>;
  using KdTree = pcl::search::KdTree<PointTarget>;
  using KdTreePtr = typename KdTree::Ptr;
  using KdTreeReciprocal = pcl::search::KdTree<PointSource>;
  using KdTreeReciprocalPtr = typename KdTreeReciprocal::Ptr;
  using PointCloudSource = pcl::PointCloud<PointSource>;
  using PointCloudSourceConstPtr = typename PointCloudSource::ConstPtr;
  using PointCloudTarget = pcl::PointCloud<PointTarget>;
  using PointCloudTargetConstPtr = typename PointCloudTarget::ConstPtr;
  using TransformationEstimation = pcl::registration::TransformationEstimation<PointSource, PointTarget, Scalar>;
  using TransformationEstimationPtr = typename TransformationEstimation::Ptr;
  using CorrespondenceEstimation = pcl::registration::CorrespondenceEstimationBase<PointSource, PointTarget, Scalar>;
  using CorrespondenceEstimationPtr = typename CorrespondenceEstimation::Ptr;  // registration.h:99-101

  Registration()
  : tree_(new KdTree), tree_reciprocal_(new KdTreeReciprocal), final_transformation_(Matrix4::Identity()),
    transformation_(Matrix4::Identity()), previous_transformation_(Matrix4::Identity()),
    euclidean_fitness_epsilon_(-std::numeric_limits<double>::max()),
    corr_dist_threshold_(std::sqrt(std::numeric_limits<double>::max()))
  {
  }
  ~Registration() override
  {
    if (icp_) pclb200_icp_destroy(icp_);
  }

  using CorrespondenceRejectorPtr = pcl::registration::CorrespondenceRejector::Ptr;
  // registration.h:373-416
  void addCorrespondenceRejector(const CorrespondenceRejectorPtr& rejector) { correspondence_rejectors_.push_back(rejector); }
  std::vector<CorrespondenceRejectorPtr> getCorrespondenceRejectors() { return correspondence_rejectors_; }
  bool removeCorrespondenceRejector(unsigned int i)
  {
    if (i >= correspondence_rejectors_.size()) return false;
    correspondence_rejectors_.erase(correspondence_rejectors_.begin() + i);
    return true;
  }
  void clearCorrespondenceRejectors() { correspondence_rejectors_.clear(); }

  // registration.h:419-425: the representation the TARGET searcher indexes with (dimensions / rescale values)
  using PointRepresentationConstPtr = typename KdTree::PointRepresentationConstPtr;
  void setPointRepresentation(const PointRepresentationConstPtr& point_representation)
  {
    point_representation_ = point_representation;
    target_cloud_updated_ = true;
  }

  void setTransformationEstimation(const TransformationEstimationPtr& te) { transformation_estimation_ = te; }
  void setCorrespondenceEstimation(const CorrespondenceEstimationPtr& ce) { correspondence_estimation_ = ce; }

  // impl/registration.hpp:47-71
  virtual void setInputSource(const PointCloudSourceConstPtr& cloud)
  {
    if (!cloud || cloud->empty()) {
      std::fprintf(stderr, "[pcl::%s::setInputSource] Invalid or empty point cloud dataset given!\n", getClassName().c_str());
      return;
    }
    source_cloud_updated_ = true;
    PCLBase<PointSource>::setInputCloud(cloud);
  }
  PointCloudSourceConstPtr const getInputSource() { return this->input_; }
  virtual void setInputTarget(const PointCloudTargetConstPtr& cloud)
  {
    if (!cloud || cloud->empty()) {
      std::fprintf(stderr, "[pcl::%s::setInputTarget] Invalid or empty point cloud dataset given!\n", getClassName().c_str());
      return;
    }
    target_ = cloud;
    target_cloud_updated_ = true;
  }
  PointCloudTargetConstPtr const getInputTarget() { return target_; }

  // registration.h:214-246
  void setSearchMethodTarget(const KdTreePtr& tree, bool force_no_recompute = false)
  {
    tree_ = tree;
    force_no_recompute_ = force_no_recompute;
    target_cloud_updated_ = true;
  }
  KdTreePtr getSearchMethodTarget() const { return tree_; }
  void setSearchMethodSource(const KdTreeReciprocalPtr& tree, bool force_no_recompute = false)
  {
    tree_reciprocal_ = tree;
    force_no_recompute_reciprocal_ = force_no_recompute;
    source_cloud_updated_ = true;
  }
  KdTreeReciprocalPtr getSearchMethodSource() const { return tree_reciprocal_; }

  Matrix4 getFinalTransformation() { return final_transformation_; }
  Matrix4 getLastIncrementalTransformation() { return transformation_; }
  void setMaximumIterations(int n) { max_iterations_ = n; }
  int getMaximumIterations() { return max_iterations_; }
  void setRANSACIterations(int n) { ransac_iterations_ = n; }
  void setRANSACOutlierRejectionThreshold(double t) { inlier_threshold_ = t; }
  int getRANSACIterations() { return ransac_iterations_; }                       // registration.h:299-304
  double getRANSACOutlierRejectionThreshold() { return inlier_threshold_; }      // registration.h:322-327
  void setMaxCorrespondenceDistance(double d) { corr_dist_threshold_ = d; }
  double getMaxCorrespondenceDistance() { return corr_dist_threshold_; }
  void setTransformationEpsilon(double e) { transformation_epsilon_ = e; }
  double getTransformationEpsilon() { return transformation_epsilon_; }
  void setTransformationRotationEpsilon(double e) { transformation_rotation_epsilon_ = e; }
  double getTransformationRotationEpsilon() { return transformation_rotation_epsilon_; }
  void setEuclideanFitnessEpsilon(double e) { euclidean_fitness_epsilon_ = e; }
  double getEuclideanFitnessEpsilon() { return euclidean_fitness_epsilon_; }
  bool hasConverged() const { return converged_; }
  const std::string& getClassName() const { return reg_name_; }

  // impl/registration.hpp:134-168
  double getFitnessScore(double max_range = std::numeric_limits<double>::max(), bool use_indices = false)
  {
    if (!tree_->deviceIndex() || !this->input_) return std::numeric_limits<double>::max();
    double T[16], score = std::numeric_limits<double>::max();
    toRowMajor(final_transformation_, T);
    const bool sub = use_indices && this->indices_ && this->indices_->size() != this->input_->size();
    int rc = pclb200_fitness_score(b200::Context::get(), tree_->deviceIndex(), this->input_->points.data(), this->input_->size(),
                                   sizeof(PointSource), sub ? this->indices_->data() : nullptr, sub ? this->indices_->size() : 0,
                                   this->input_->is_dense ? 1 : 0, T, sizeof(Scalar) == 8, max_range, &score);
    if (rc != PCLB200_OK) std::fprintf(stderr, "[pcl::%s::getFitnessScore] %s\n", getClassName().c_str(), pclb200_last_error());
    return score;
  }

  // getFitnessScore(distances_a, distances_b) — impl/registration.hpp:105-130
  double getFitnessScore(const std::vector<float>& distances_a, const std::vector<float>& distances_b)
  {
    const unsigned int nr = static_cast<unsigned int>(std::min(distances_a.size(), distances_b.size()));
    double sum = 0.0;
    for (unsigned int i = 0; i < nr; ++i) sum += static_cast<double>(distances_a[i]) - static_cast<double>(distances_b[i]);
    return nr ? std::abs(sum / nr) : 0.0;
  }
  // registration.h:431-442: called after every iteration with the transformed source and the correspondences
  using UpdateVisualizerCallbackSignature = void(const pcl::PointCloud<PointSource>&, const pcl::Indices&,
                                                 const pcl::PointCloud<PointTarget>&, const pcl::Indices&);
  bool registerVisualizationCallback(std::function<UpdateVisualizerCallbackSignature>& cb)
  {
    if (cb) { update_visualizer_ = cb; return true; }
    return false;
  }

  // impl/registration.hpp:172-221
  void align(PointCloudSource& output) { align(output, Matrix4::Identity()); }
  void align(PointCloudSource& output, const Matrix4& guess)
  {
    if (!initCompute()) return;
    output.resize(this->indices_->size());
    output.header = this->input_->header;
    if (this->indices_->size() != this->input_->size()) {
      output.width = static_cast<std::uint32_t>(this->indices_->size());
      output.height = 1;
    }
    else {
      output.width = this->input_->width;
      output.height = this->input_->height;
    }
    output.is_dense = this->input_->is_dense;
    converged_ = false;
    final_transformation_ = transformation_ = previous_transformation_ = Matrix4::Identity();
    computeTransformation(output, guess);
    this->deinitCompute();
  }

protected:
  // impl/registration.hpp:73-101
  bool initCompute()
  {
    if (!target_) {
      std::fprintf(stderr, "[pcl::registration::%s::compute] No input target dataset was given!\n", getClassName().c_str());
      return false;
    }
    if (target_cloud_updated_ && !force_no_recompute_) {
      if (point_representation_)  // impl/registration.hpp:84-91
        tree_->setPointRepresentation(point_representation_);
      tree_->setInputCloud(target_);
      target_cloud_updated_ = false;
      target_uploaded_ = false;
    }
    return PCLBase<PointSource>::initCompute();
  }
  virtual void computeTransformation(PointCloudSource& output, const Matrix4& guess) = 0;

  static void toRowMajor(const Matrix4& M, double* t)
  {
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) t[4 * r + c] = static_cast<double>(M(r, c));
  }
  static void fromRowMajor(const double* t, Matrix4& M)
  {
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) M(r, c) = static_cast<Scalar>(t[4 * r + c]);
  }

  std::string reg_name_ = "Registration";
  KdTreePtr tree_;
  KdTreeReciprocalPtr tree_reciprocal_;
  int nr_iterations_ = 0;
  int max_iterations_ = 10;  // registration.h:566
  int ransac_iterations_ = 0;
  PointCloudTargetConstPtr target_;
  Matrix4 final_transformation_, transformation_, previous_transformation_;
  double transformation_epsilon_ = 0.0;           // :588
  double transformation_rotation_epsilon_ = 0.0;
  double euclidean_fitness_epsilon_;              // :116
  double corr_dist_threshold_;                    // :117
  double inlier_threshold_ = 0.05;
  bool converged_ = false;
  CorrespondenceEstimationPtr correspondence_estimation_;
  TransformationEstimationPtr transformation_estimation_;
  std::vector<CorrespondenceRejectorPtr> correspondence_rejectors_;
  bool target_cloud_updated_ = true, source_cloud_updated_ = true;
  bool force_no_recompute_ = false, force_no_recompute_reciprocal_ = false;
  bool target_uploaded_ = false;
  PointRepresentationConstPtr point_representation_;
  pclb200_icp* icp_ = nullptr;
  std::function<UpdateVisualizerCallbackSignature> update_visualizer_;
};

template <typename PointSource, typename PointTarget, typename Scalar = float>
class IterativeClosestPoint : public Registration<PointSource, PointTarget, Scalar> {
public:
  using Base = Registration<PointSource, PointTarget, Scalar>;
  using Matrix4 = typename Base::Matrix4;
  using Ptr = std::shared_ptr<IterativeClosestPoint>;
  using PointCloudSource = typename Base::PointCloudSource;
  using ConvergenceCriteria = pcl::registration::DefaultConvergenceCriteria<Scalar>;

  IterativeClosestPoint() : convergence_criteria_(new ConvergenceCriteria)
  {
    this->reg_name_ = "IterativeClosestPoint";
    this->transformation_estimation_.reset(new pcl::registration::TransformationEstimationSVD<PointSource, PointTarget, Scalar>());
    this->correspondence_estimation_.reset(new pcl::registration::CorrespondenceEstimation<PointSource, PointTarget, Scalar>());
  }
  typename ConvergenceCriteria::Ptr getConvergeCriteria() { return convergence_criteria_; }
  void setUseReciprocalCorrespondences(bool v) { use_reciprocal_correspondence_ = v; }
  bool getUseReciprocalCorrespondences() const { return use_reciprocal_correspondence_; }
  void setNumberOfThreads(unsigned int) {}
  int getNumberOfIterations() const { return this->nr_iterations_; }
  std::int64_t getNumberOfCorrespondences() const { return n_correspondences_; }

protected:
  virtual bool withNormalsTransform() const { return false; }
  virtual bool enforceSameDirectionNormals() const { return true; }

  // ---- the reference's loop, stage by stage, for searchers that index representation vectors --------------------------
  // With a non-trivial PointRepresentation (dimensions dropped, per-dimension rescale) the correspondence search runs in
  // the representation's space while the transform is estimated on the real coordinates (impl/icp.hpp:164-241).  The
  // fused device loop searches raw xyz, so this case runs the reference's own structure: batch 1-NN through the
  // searcher (one device launch), gate, rejector chain, estimator (device), transformCloud, convergence criteria.
  static void transformCloudHost(const PointCloudSource& in, PointCloudSource& out, const Matrix4& T)
  {
    float tr[12];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 4; ++c) tr[4 * r + c] = static_cast<float>(T(r, c));
    if (&in != &out) out = in;
    for (auto& p : out.points) {  // impl/icp.hpp:49-111 (fp32, left to right; non-finite points untouched)
      if (!isXYZFinite(p)) continue;
      const float x = p.x, y = p.y, z = p.z;
      p.x = ((tr[0] * x + tr[1] * y) + tr[2] * z) + tr[3];
      p.y = ((tr[4] * x + tr[5] * y) + tr[6] * z) + tr[7];
      p.z = ((tr[8] * x + tr[9] * y) + tr[10] * z) + tr[11];
    }
  }
  // icp.hpp:157-161: the criteria object takes Registration's thresholds; the rotation threshold only when one was set
  void syncConvergenceCriteria()
  {
    auto& cc = *convergence_criteria_;
    cc.max_iterations_ = this->max_iterations_;
    cc.mse_threshold_relative_ = this->euclidean_fitness_epsilon_;
    cc.translation_threshold_ = this->transformation_epsilon_;
    if (this->transformation_rotation_epsilon_ > 0) cc.rotation_threshold_ = this->transformation_rotation_epsilon_;
  }

  void computeTransformationStaged(PointCloudSource& output, const Matrix4& guess)
  {
    using State = typename ConvergenceCriteria::ConvergenceState;
    syncConvergenceCriteria();
    PointCloudSource moved = *this->input_;
    this->nr_iterations_ = 0;
    this->converged_ = false;
    this->final_transformation_ = guess;
    if (!(guess == Matrix4::Identity())) transformCloudHost(*this->input_, moved, guess);  // impl/icp.hpp:125-134
    this->transformation_ = Matrix4::Identity();
    State state = ConvergenceCriteria::CONVERGENCE_CRITERIA_NOT_CONVERGED;
    double& prev_mse = convergence_criteria_->prev_mse_;
    int iterations_similar = 0;
    const double max_d2 = this->corr_dist_threshold_ * this->corr_dist_threshold_;
    pcl::Correspondences corr, tmp;
    {  // impl/icp.hpp:142-155: rejectors that ask for the target cloud get it once, as a blob
      pcl::PCLPointCloud2::Ptr target_blob;
      for (const auto& rej : this->correspondence_rejectors_)
        if (rej->requiresTargetPoints()) {
          if (!target_blob) { target_blob.reset(new pcl::PCLPointCloud2); pcl::toPCLPointCloud2(*this->target_, *target_blob); }
          rej->setTargetPoints(target_blob);
        }
    }
    do {
      this->previous_transformation_ = this->transformation_;
      // correspondences (impl/correspondence_estimation.hpp:145-218): one batch 1-NN for all source indices
      std::vector<Indices> ki;
      std::vector<std::vector<float>> kd;
      {
        pcl::PointCloud<PointTarget> q;
        q.points.reserve(this->indices_->size());
        for (index_t i : *this->indices_) {
          PointTarget t;
          t.x = moved[i].x; t.y = moved[i].y; t.z = moved[i].z;
          q.points.push_back(t);
        }
        this->tree_->nearestKSearch(q, Indices(), 1, ki, kd);
      }
      corr.clear();
      for (std::size_t j = 0; j < this->indices_->size(); ++j) {
        const index_t i = (*this->indices_)[j];
        if (!this->input_->is_dense && !isXYZFinite(moved[i])) continue;
        if (ki[j].empty() || static_cast<double>(kd[j][0]) > max_d2) continue;
        corr.emplace_back(i, ki[j][0], kd[j][0]);
      }
      {
        pcl::PCLPointCloud2::Ptr moved_blob;  // impl/icp.hpp:166-170, 191-192: the transformed source of THIS iteration
        for (const auto& rej : this->correspondence_rejectors_) {  // impl/icp.hpp:187-201
          if (rej->requiresSourcePoints()) {
            if (!moved_blob) { moved_blob.reset(new pcl::PCLPointCloud2); pcl::toPCLPointCloud2(moved, *moved_blob); }
            rej->setSourcePoints(moved_blob);
          }
          rej->getRemainingCorrespondences(corr, tmp);
          corr.swap(tmp);
        }
      }
      if (corr.size() < 3) {  // impl/icp.hpp:204-213
        std::fprintf(stderr, "[pcl::%s::computeTransformation] Not enough correspondences found. Relax your threshold parameters.\n",
                     this->getClassName().c_str());
        state = ConvergenceCriteria::CONVERGENCE_CRITERIA_NO_CORRESPONDENCES;
        this->converged_ = false;
        break;
      }
      this->transformation_estimation_->estimateRigidTransformation(moved, *this->target_, corr, this->transformation_);
      transformCloudHost(moved, moved, this->transformation_);
      this->final_transformation_ = this->transformation_ * this->final_transformation_;
      ++this->nr_iterations_;
      n_correspondences_ = static_cast<std::int64_t>(corr.size());
      // DefaultConvergenceCriteria::hasConverged — impl/default_convergence_criteria.hpp:49-140
      {
        if (state != ConvergenceCriteria::CONVERGENCE_CRITERIA_NOT_CONVERGED) {
          iterations_similar = 0;
          state = ConvergenceCriteria::CONVERGENCE_CRITERIA_NOT_CONVERGED;
        }
        bool conv = false, similar = false;
        const auto& cc = *convergence_criteria_;
        if (this->nr_iterations_ >= this->max_iterations_) {
          if (!cc.failure_after_max_iter_) { state = ConvergenceCriteria::CONVERGENCE_CRITERIA_ITERATIONS; conv = true; }
          else state = ConvergenceCriteria::CONVERGENCE_CRITERIA_FAILURE_AFTER_MAX_ITERATIONS;
        }
        if (!conv) {
          const Matrix4& T = this->transformation_;
          const double cos_angle = 0.5 * (T(0, 0) + T(1, 1) + T(2, 2) - 1);
          const double t2 = T(0, 3) * T(0, 3) + T(1, 3) * T(1, 3) + T(2, 3) * T(2, 3);
          const double rot_thr = cc.rotation_threshold_;
          double mse = 0.0;
          for (const auto& c : corr) mse += c.distance;
          mse /= static_cast<double>(corr.size());
          auto hit = [&](State s2) {
            if (iterations_similar >= cc.max_iterations_similar_transforms_) { state = s2; conv = true; }
            else similar = true;
          };
          if (cos_angle >= rot_thr && t2 <= this->transformation_epsilon_) hit(ConvergenceCriteria::CONVERGENCE_CRITERIA_TRANSFORM);
          if (!conv && std::abs(mse - prev_mse) < cc.mse_threshold_absolute_) hit(ConvergenceCriteria::CONVERGENCE_CRITERIA_ABS_MSE);
          if (!conv && std::abs(mse - prev_mse) / prev_mse < this->euclidean_fitness_epsilon_) hit(ConvergenceCriteria::CONVERGENCE_CRITERIA_REL_MSE);
          if (!conv) {
            iterations_similar = similar ? iterations_similar + 1 : 0;
            prev_mse = mse;
          }
        }
        this->converged_ = conv;
      }
    } while (!this->converged_ && state != ConvergenceCriteria::CONVERGENCE_CRITERIA_FAILURE_AFTER_MAX_ITERATIONS);
    convergence_criteria_->state_ = state;
    transformCloudHost(*this->input_, output, this->final_transformation_);  // impl/icp.hpp:265-267
  }

  // impl/icp.hpp:113-268 — the whole do-while runs on the device; the host only evaluates the convergence criteria
  void computeTransformation(PointCloudSource& output, const Matrix4& guess) override
  {
    bool host_rejector = false;
    for (const auto& r : this->correspondence_rejectors_) host_rejector = host_rejector || !r->runsOnDevice();
    if (this->tree_->usesRepresentationVectors() || host_rejector) {
      computeTransformationStaged(output, guess);
      return;
    }
    syncConvergenceCriteria();
    pclb200_ctx* ctx = b200::Context::get();
    pclb200_icp_params P;
    pclb200_icp_default_params(&P);
    P.max_iterations = this->max_iterations_;
    P.use_reciprocal = use_reciprocal_correspondence_ ? 1 : 0;
    P.estimator = this->transformation_estimation_->abiEstimator();
    if (auto* svd = dynamic_cast<const registration::TransformationEstimationSVD<PointSource, PointTarget, Scalar>*>(
            this->transformation_estimation_.get()))
      P.svd_no_umeyama = svd->usesUmeyama() ? 0 : 1;  // TransformationEstimationSVD(false): the correlation formula
    P.scalar_is_double = sizeof(Scalar) == 8;
    P.with_normals_transform = withNormalsTransform() ? 1 : 0;
    P.is_dense = this->input_->is_dense ? 1 : 0;
    P.enforce_same_direction_normals = enforceSameDirectionNormals() ? 1 : 0;
    P.failure_after_max_iter = convergence_criteria_->failure_after_max_iter_ ? 1 : 0;
    P.max_iterations_similar_transforms = convergence_criteria_->max_iterations_similar_transforms_;
    P.max_correspondence_distance = this->corr_dist_threshold_;
    P.transformation_epsilon = this->transformation_epsilon_;
    // a threshold set on the criteria object is honoured: the library takes any value > 0 as the cos-angle threshold
    P.transformation_rotation_epsilon = convergence_criteria_->rotation_threshold_ > 0
                                            ? convergence_criteria_->rotation_threshold_
                                            : this->transformation_rotation_epsilon_;
    P.euclidean_fitness_epsilon = this->euclidean_fitness_epsilon_;
    P.mse_threshold_absolute = convergence_criteria_->mse_threshold_absolute_;
    // setCorrespondenceEstimation(NormalShooting / BackProjection): the fused loop runs that estimator, on the normal
    // fields of the two clouds (what icp.hpp:166-180 hands over as blobs)
    P.correspondence_kind = this->correspondence_estimation_->abiKind();
    P.correspondence_k = this->correspondence_estimation_->abiK();
    this->nr_iterations_ = 0;
    this->converged_ = false;
    this->final_transformation_ = guess;
    auto fail = [&](const char* where) {
      std::fprintf(stderr, "[pcl::%s::computeTransformation] %s: %s\n", this->getClassName().c_str(), where, pclb200_last_error());
    };
    if (!this->tree_->deviceIndex()) { fail("target index"); return; }
    if (!this->icp_) {
      if (pclb200_icp_create(ctx, &P, &this->icp_) != PCLB200_OK) { fail("icp_create"); return; }
      this->target_uploaded_ = false;
    }
    else if (pclb200_icp_set_params(this->icp_, &P) != PCLB200_OK) { fail("icp_set_params"); return; }
    if (!this->target_uploaded_ || uploaded_index_ != this->tree_->deviceIndex()) {
      const void* tn = nullptr;
      if (has_normal<PointTarget>::value && !this->target_->empty())
        tn = reinterpret_cast<const unsigned char*>(this->target_->points.data()) + 16;  // normal_x of point 0
      if (pclb200_icp_set_target(this->icp_, this->tree_->deviceIndex(), tn, sizeof(PointTarget)) != PCLB200_OK) { fail("icp_set_target"); return; }
      this->target_uploaded_ = true;
      uploaded_index_ = this->tree_->deviceIndex();
    }
    {
      std::vector<pclb200_rejector> chain;
      for (const auto& r : this->correspondence_rejectors_) chain.push_back(r->abiRejector());
      if (pclb200_icp_set_rejectors(this->icp_, chain.data(), static_cast<int>(chain.size())) != PCLB200_OK) { fail("icp_set_rejectors"); return; }
    }
    double g[16];
    Base::toRowMajor(guess, g);
    const void* sn = nullptr;
    if (has_normal<PointSource>::value)
      sn = reinterpret_cast<const unsigned char*>(this->input_->points.data()) + 16;
    if (pclb200_icp_set_source(this->icp_, this->input_->points.data(), this->input_->size(), sizeof(PointSource), sn, sizeof(PointSource),
                               this->abiIndices(), this->abiIndexCount(), guess == Matrix4::Identity() ? nullptr : g) != PCLB200_OK) {
      fail("icp_set_source");
      return;
    }
    pclb200_icp_stats st;
    if (!this->update_visualizer_) {
      if (pclb200_icp_iterate(this->icp_, std::numeric_limits<int>::max(), &st) != PCLB200_OK) { fail("icp_iterate"); return; }
    }
    else {
      // icp.hpp:228-236: one iteration at a time so the callback sees every intermediate state
      pcl::Correspondences corr;
      PointCloudSource moved;
      do {
        if (pclb200_icp_iterate(this->icp_, 1, &st) != PCLB200_OK) { fail("icp_iterate"); return; }
        if (st.state == PCLB200_CONV_NO_CORRESPONDENCES) break;
        corr.resize(this->indices_->size());
        std::size_t nc = 0;
        if (pclb200_icp_get_correspondences(this->icp_, reinterpret_cast<pclb200_corr*>(corr.data()), &nc) != PCLB200_OK) { fail("icp_get_correspondences"); return; }
        corr.resize(nc);
        moved = *this->input_;
        void* mn = has_normal<PointSource>::value ? reinterpret_cast<unsigned char*>(moved.points.data()) + 16 : nullptr;
        if (pclb200_icp_get_cloud(this->icp_, moved.points.data(), sizeof(PointSource), mn, sizeof(PointSource)) != PCLB200_OK) { fail("icp_get_cloud"); return; }
        pcl::Indices si, ti;
        for (const auto& c : corr) { si.push_back(c.index_query); ti.push_back(c.index_match); }
        this->update_visualizer_(moved, si, *this->target_, ti);
      } while (st.state == PCLB200_CONV_NOT_CONVERGED);
    }
    Base::fromRowMajor(st.final_transformation, this->final_transformation_);
    Base::fromRowMajor(st.last_transformation, this->transformation_);
    this->previous_transformation_ = this->transformation_;
    this->nr_iterations_ = st.iterations;
    this->converged_ = st.converged != 0;
    n_correspondences_ = st.n_correspondences;
    convergence_criteria_->state_ = static_cast<typename ConvergenceCriteria::ConvergenceState>(st.state);
    if (st.state == PCLB200_CONV_NO_CORRESPONDENCES)
      std::fprintf(stderr, "[pcl::%s::computeTransformation] Not enough correspondences found. Relax your threshold parameters.\n",
                   this->getClassName().c_str());
    // output = *input_, transformed by final_transformation_ (icp.hpp:265-267)
    output = *this->input_;
    void* on = has_normal<PointSource>::value ? reinterpret_cast<unsigned char*>(output.points.data()) + 16 : nullptr;
    if (pclb200_icp_get_cloud(this->icp_, output.points.data(), sizeof(PointSource), on, sizeof(PointSource)) != PCLB200_OK)
      fail("icp_get_cloud");
  }

  typename ConvergenceCriteria::Ptr convergence_criteria_;
  bool use_reciprocal_correspondence_ = false;
  std::int64_t n_correspondences_ = 0;
  pclb200_index* uploaded_index_ = nullptr;
};

// icp.h:339-456 — point-to-plane variant (non-symmetric objective)
template <typename PointSource, typename PointTarget, typename Scalar = float>
class IterativeClosestPointWithNormals : public IterativeClosestPoint<PointSource, PointTarget, Scalar> {
public:
  using Ptr = std::shared_ptr<IterativeClosestPointWithNormals>;
  IterativeClosestPointWithNormals()
  {
    this->reg_name_ = "IterativeClosestPointWithNormals";
    setUseSymmetricObjective(false);          // icp.h:366-371
    setEnforceSameDirectionNormals(true);
  }
  // icp.h:381-418
  void setUseSymmetricObjective(bool symmetric) { use_symmetric_objective_ = symmetric; resetEstimator(); }
  bool getUseSymmetricObjective() const { return use_symmetric_objective_; }
  void setEnforceSameDirectionNormals(bool v) { enforce_same_direction_normals_ = v; resetEstimator(); }
  bool getEnforceSameDirectionNormals() const { return enforce_same_direction_normals_; }

protected:
  bool withNormalsTransform() const override { return true; }  // impl/icp.hpp:312-318
  bool enforceSameDirectionNormals() const override { return enforce_same_direction_normals_; }
  template <typename PS = PointSource>
  typename std::enable_if<has_normal<PS>::value>::type makeSymmetric()
  {
    auto est = std::make_shared<pcl::registration::TransformationEstimationSymmetricPointToPlaneLLS<PointSource, PointTarget, Scalar>>();
    est->setEnforceSameDirectionNormals(enforce_same_direction_normals_);
    this->transformation_estimation_ = est;
  }
  template <typename PS = PointSource>
  typename std::enable_if<!has_normal<PS>::value>::type makeSymmetric()
  {
    std::fprintf(stderr, "[pcl::IterativeClosestPointWithNormals] the symmetric objective needs source normals\n");
  }
  void resetEstimator()
  {
    if (use_symmetric_objective_)
      makeSymmetric();
    else
      this->transformation_estimation_.reset(new pcl::registration::TransformationEstimationPointToPlaneLLS<PointSource, PointTarget, Scalar>());
  }
  bool use_symmetric_objective_ = false;
  bool enforce_same_direction_normals_ = true;
};

}  // namespace pcl
