#include "dataset.h"

#include "../../../include/gpboost_b200_dev.h"
#include "runtime.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <limits>
#include <unordered_set>
#include <sstream>
#include <stdexcept>

namespace gpb200 {

namespace {
constexpr double kZeroThreshold = 1e-35f;  // the reference's zero band (include/LightGBM/meta.h:56): |v| <= this is "zero"
[[noreturn]] void Fatal(const std::string& m) { throw std::runtime_error(m); }

// ---- row sample --------------------------------------------------------------------------------------------------
// The bin boundaries are a function of WHICH rows are sampled, so the sampler has to draw the reference's rows: the
// 32-bit multiplicative congruential stream of include/LightGBM/utils/random.h (x <- 214013 x + 2531011; 15 bits from
// bit 16 for the float draw, the low 31 bits for the integer draw) and its three regimes (everything / one Bernoulli draw
// per row when the sample is a large part of the data / Floyd's subset algorithm otherwise), ascending row ids.
struct SampleStream {
  uint32_t state;
  uint32_t Advance() { state = state * 214013u + 2531011u; return state; }
  float Unit() { return static_cast<float>((Advance() >> 16) & 0x7FFFu) / 32768.0f; }
  int Below(int bound) { return static_cast<int>(Advance() & 0x7FFFFFFFu) % bound; }
};

std::vector<int> DrawSampleRows(int num_rows, int want, int seed) {
  std::vector<int> rows;
  if (want <= 0 || want > num_rows) return rows;
  SampleStream rng{static_cast<uint32_t>(seed)};
  rows.reserve(want);
  if (want == num_rows) {
    rows.resize(num_rows);
    for (int i = 0; i < num_rows; ++i) rows[i] = i;
    return rows;
  }
  if (want > 1 && want > num_rows / std::log2(want)) {
    // selection sampling: row i is taken with probability (still wanted) / (still available)
    for (int i = 0; i < num_rows; ++i) {
      const double p_take = (want - rows.size()) / static_cast<double>(num_rows - i);
      if (rng.Unit() < p_take) rows.push_back(i);
    }
    return rows;
  }
  // Floyd: for r = N-K .. N-1 draw v in [0, r); take v unless already taken, else take r
  std::unordered_set<int> taken;
  taken.reserve(2 * want);
  for (int r = num_rows - want; r < num_rows; ++r) {
    const int v = rng.Below(r);
    rows.push_back(taken.insert(v).second ? v : (taken.insert(r), r));
  }
  std::sort(rows.begin(), rows.end());
  return rows;
}

// ---- bin boundaries ----------------------------------------------------------------------------------------------
// What has to come out (BinMapper::FindBin for a numerical feature without NaNs, src/LightGBM/io/bin.cpp:325-520 with
// FindBinWithZeroAsOneBin :241-297 and GreedyFindBin :78-155): the strictly increasing upper bounds b_0 < ... < b_{k-1} = +inf with
// zero in a bin of its own. Formulated here on a run-length view of the sorted sample:
//   * Runs: maximal groups of sample values that are equal up to one ulp, represented by their largest member, with an explicit
//     run for the implicit zeros (rows whose |value| is inside the zero band are not part of the sample vector);
//   * a side (the negative runs, or the positive runs) is cut into at most `budget` bins by CutSide(), which returns the run
//     indices after which a bin ends; a bound is the midpoint between the last run of a bin and the first run of the next one,
//     nudged one ulp up, and dropped when it does not exceed the previous bound by more than an ulp.
struct Run { double value; int count; };

inline double UlpUp(double a) { return std::nextafter(a, std::numeric_limits<double>::infinity()); }
inline bool WithinUlp(double lo, double hi) { return hi <= UlpUp(lo); }  // for lo <= hi

std::vector<Run> BuildRuns(std::vector<double>& sample, int implicit_zeros) {
  std::stable_sort(sample.begin(), sample.end());
  std::vector<Run> runs;
  const size_t ns = sample.size();
  if (ns == 0 || (sample[0] > 0.0 && implicit_zeros > 0)) runs.push_back({0.0, implicit_zeros});
  for (size_t i = 0; i < ns; ++i) {
    if (i > 0 && WithinUlp(sample[i - 1], sample[i])) {
      runs.back().value = sample[i];
      ++runs.back().count;
      continue;
    }
    if (i > 0 && sample[i - 1] < 0.0 && sample[i] > 0.0) runs.push_back({0.0, implicit_zeros});  // zero sits between the signs
    runs.push_back({sample[i], 1});
  }
  if (ns > 0 && sample[ns - 1] < 0.0 && implicit_zeros > 0) runs.push_back({0.0, implicit_zeros});
  return runs;
}

// Appends midpoint bounds; keeps the list strictly increasing by more than an ulp.
struct BoundList {
  std::vector<double> b;
  void Between(double last_of_bin, double first_of_next) {
    const double cut = UlpUp((last_of_bin + first_of_next) / 2.0);
    if (b.empty() || !WithinUlp(b.back(), cut)) b.push_back(cut);
  }
};

// Bins for runs[0..nr): at most `budget` of them, at least `min_in_bin` sample rows each where possible; `rows` = sample rows on
// this side. Returns the bounds, the last one +inf.
std::vector<double> CutSide(const Run* runs, int nr, int budget, int64_t rows, int min_in_bin) {
  if (budget <= 0) Fatal("Check failed: max_bin > 0");
  BoundList out;
  if (nr <= budget) {
    // few distinct values: every run may get its own bin as soon as the bin holds min_in_bin rows
    int held = 0;
    for (int i = 0; i + 1 < nr; ++i) {
      held += runs[i].count;
      if (held < min_in_bin) continue;
      const size_t before = out.b.size();
      out.Between(runs[i].value, runs[i + 1].value);
      if (out.b.size() != before) held = 0;
    }
    out.b.push_back(std::numeric_limits<double>::infinity());
    return out.b;
  }
  if (min_in_bin > 0) budget = std::max(1, std::min(budget, static_cast<int>(rows / min_in_bin)));
  // equal-frequency cutting; runs at least as heavy as the average bin get a bin of their own and leave the average
  double target = static_cast<double>(rows) / budget;
  std::vector<char> heavy(nr, 0);
  int light_bins = budget;
  int light_rows = static_cast<int>(rows);
  for (int i = 0; i < nr; ++i) {
    if (runs[i].count >= target) { heavy[i] = 1; --light_bins; light_rows -= runs[i].count; }
  }
  target = static_cast<double>(light_rows) / light_bins;
  std::vector<int> cut_after;  // run index that closes a bin
  int held = 0;
  for (int i = 0; i + 1 < nr; ++i) {
    if (!heavy[i]) light_rows -= runs[i].count;
    held += runs[i].count;
    const bool close = heavy[i] || held >= target || (heavy[i + 1] && held >= std::max(1.0, target * 0.5f));
    if (!close) continue;
    cut_after.push_back(i);
    if (static_cast<int>(cut_after.size()) >= budget - 1) break;
    held = 0;
    if (!heavy[i]) { --light_bins; target = light_rows / static_cast<double>(light_bins); }
  }
  for (int i : cut_after) out.Between(runs[i].value, runs[i + 1].value);
  out.b.push_back(std::numeric_limits<double>::infinity());
  return out.b;
}

// true when no bound leaves at least `need` sample rows on both sides (the feature cannot be split: bin.cpp:53-66)
bool NoUsefulCut(const std::vector<int>& rows_in_bin, int total, int need) {
  int left = 0;
  for (size_t i = 0; i + 1 < rows_in_bin.size(); ++i) {
    left += rows_in_bin[i];
    if (left >= need && total - left >= need) return false;
  }
  return true;
}

FeatureBins BoundsFromSample(std::vector<double>& sample, size_t sample_rows, int max_bin, int min_in_bin, int min_split_rows, bool pre_filter) {
  for (double v : sample)
    if (std::isnan(v)) Fatal("Missing values (NaN) in the feature matrix are not supported by the CUDA tree learner yet");
  FeatureBins fb;
  const std::vector<Run> runs = BuildRuns(sample, static_cast<int>(sample_rows - sample.size()));
  const int nr = static_cast<int>(runs.size());
  fb.min_val = runs.front().value;
  fb.max_val = runs.back().value;
  // sides: [0, neg_end) negative, [pos_begin, nr) positive, anything between is the zero run
  int neg_end = 0, pos_begin = nr;
  int64_t neg_rows = 0, pos_rows = 0, zero_rows = 0;
  while (neg_end < nr && runs[neg_end].value <= -kZeroThreshold) neg_rows += runs[neg_end++].count;
  for (int i = neg_end; i < nr; ++i) {
    if (runs[i].value > kZeroThreshold) { if (pos_begin == nr) pos_begin = i; pos_rows += runs[i].count; }
    else zero_rows += runs[i].count;
  }
  std::vector<double>& ub = fb.upper_bounds;
  if (neg_end > 0 && max_bin > 1) {
    const int share = static_cast<int>(static_cast<double>(neg_rows) / (sample_rows - zero_rows) * (max_bin - 1));
    ub = CutSide(runs.data(), neg_end, std::max(1, share), neg_rows, min_in_bin);
    if (!ub.empty()) ub.back() = -kZeroThreshold;  // the negative side ends where the zero bin starts
  }
  const int pos_budget = max_bin - 1 - static_cast<int>(ub.size());
  if (pos_begin < nr && pos_budget > 0) {
    const std::vector<double> pos = CutSide(runs.data() + pos_begin, nr - pos_begin, pos_budget, pos_rows, min_in_bin);
    ub.push_back(kZeroThreshold);
    ub.insert(ub.end(), pos.begin(), pos.end());
  } else {
    ub.push_back(std::numeric_limits<double>::infinity());
  }
  if (ub.size() > static_cast<size_t>(max_bin)) Fatal("Check failed: bin_upper_bound.size() <= max_bin");
  fb.num_bin = static_cast<int>(ub.size());
  std::vector<int> rows_in_bin(fb.num_bin, 0);
  for (int i = 0, bin = 0; i < nr; ++i) {
    if (runs[i].value > ub[bin]) ++bin;
    rows_in_bin[bin] += runs[i].count;
  }
  fb.trivial = fb.num_bin <= 1 || (pre_filter && NoUsefulCut(rows_in_bin, static_cast<int>(sample_rows), min_split_rows));
  return fb;
}

template <typename T>
inline double At(const void* data, int32_t nrow, int32_t ncol, int is_row_major, int64_t i, int j) {
  const T* p = static_cast<const T*>(data);
  return is_row_major ? (double)p[i * ncol + j] : (double)p[(int64_t)j * nrow + i];
}

}  // namespace

// Aliases of the parameters this build reads or has to refuse (the reference resolves them in Config::alias_table,
// src/LightGBM/io/config_auto.cpp:11-170, before anything else looks at a key): alias -> canonical name.
static const std::map<std::string, std::string>& AliasTable() {
  static const std::map<std::string, std::string> t = {
      {"objective_type", "objective"}, {"app", "objective"}, {"application", "objective"}, {"likelihood", "objective"},
      {"shrinkage_rate", "learning_rate"}, {"eta", "learning_rate"},
      {"num_leaf", "num_leaves"}, {"max_leaves", "num_leaves"}, {"max_leaf", "num_leaves"},
      {"tree", "tree_learner"}, {"tree_type", "tree_learner"}, {"tree_learner_type", "tree_learner"},
      {"boosting_type", "boosting"}, {"boost", "boosting"},
      {"min_data_per_leaf", "min_data_in_leaf"}, {"min_data", "min_data_in_leaf"}, {"min_child_samples", "min_data_in_leaf"},
      {"min_sum_hessian_per_leaf", "min_sum_hessian_in_leaf"}, {"min_sum_hessian", "min_sum_hessian_in_leaf"},
      {"min_hessian", "min_sum_hessian_in_leaf"}, {"min_child_weight", "min_sum_hessian_in_leaf"},
      {"sub_row", "bagging_fraction"}, {"subsample", "bagging_fraction"}, {"bagging", "bagging_fraction"},
      {"pos_sub_row", "pos_bagging_fraction"}, {"pos_subsample", "pos_bagging_fraction"}, {"pos_bagging", "pos_bagging_fraction"},
      {"neg_sub_row", "neg_bagging_fraction"}, {"neg_subsample", "neg_bagging_fraction"}, {"neg_bagging", "neg_bagging_fraction"},
      {"subsample_freq", "bagging_freq"},
      {"sub_feature", "feature_fraction"}, {"colsample_bytree", "feature_fraction"},
      {"sub_feature_bynode", "feature_fraction_bynode"}, {"colsample_bynode", "feature_fraction_bynode"},
      {"max_tree_output", "max_delta_step"}, {"max_leaf_output", "max_delta_step"},
      {"reg_alpha", "lambda_l1"}, {"reg_lambda", "lambda_l2"}, {"lambda", "lambda_l2"},
      {"min_split_gain", "min_gain_to_split"},
      {"mc", "monotone_constraints"}, {"monotone_constraint", "monotone_constraints"},
      {"feature_contrib", "feature_contri"}, {"fc", "feature_contri"}, {"fp", "feature_contri"}, {"feature_penalty", "feature_contri"},
      {"fs", "forcedsplits_filename"}, {"forced_splits_filename", "forcedsplits_filename"}, {"forced_splits_file", "forcedsplits_filename"},
      {"forced_splits", "forcedsplits_filename"},
      {"verbose", "verbosity"},
      {"subsample_for_bin", "bin_construct_sample_cnt"}, {"data_seed", "data_random_seed"},
      {"cat_feature", "categorical_feature"}, {"categorical_column", "categorical_feature"}, {"cat_column", "categorical_feature"},
      {"num_classes", "num_class"}, {"unbalance", "is_unbalance"}, {"unbalanced_sets", "is_unbalance"},
      {"metrics", "metric"}, {"metric_types", "metric"},
  };
  return t;
}

Params Params::Parse(const char* s) {
  Params p;
  if (!s) return p;
  std::istringstream is(s);
  std::string tok;
  while (is >> tok) {
    auto eq = tok.find('=');
    if (eq == std::string::npos) continue;
    std::string key = tok.substr(0, eq);
    auto al = AliasTable().find(key);
    if (al != AliasTable().end()) key = al->second;
    p.kv[key] = tok.substr(eq + 1);
  }
  return p;
}

// Parameters that change the model in the reference but that this build does not implement: refuse them instead of training a
// different model silently. Keys are canonical (Parse resolves aliases). A value equal to the reference's default passes.
void Params::RejectUnsupported(const char* where) const {
  auto bad = [&](const std::string& k, const std::string& why) {
    Fatal(std::string(where) + ": parameter '" + k + "=" + kv.at(k) + "' is not supported by this build (" + why + ")");
  };
  auto has = [&](const char* k) { return kv.find(k) != kv.end() && !kv.at(k).empty(); };
  auto num = [&](const char* k, double d) { return has(k) ? std::stod(kv.at(k)) : d; };
  auto flag = [&](const char* k) { return has(k) && GetBool(k, false); };
  auto nonempty_list = [&](const char* k) { return has(k) && kv.at(k) != "\"\"" && kv.at(k) != "''" && kv.at(k) != "none" && kv.at(k) != "None"; };
  if (has("boosting") && kv.at("boosting") != "gbdt" && kv.at("boosting") != "gbrt") bad("boosting", "only gbdt");
  if (has("tree_learner") && kv.at("tree_learner") != "serial" && kv.at("tree_learner") != "data" && kv.at("tree_learner") != "data_parallel")
    bad("tree_learner", "serial, or data-parallel through GPB200_NcclInit");
  for (const char* k : {"bagging_fraction", "pos_bagging_fraction", "neg_bagging_fraction", "feature_fraction", "feature_fraction_bynode"})
    if (num(k, 1.0) < 1.0) bad(k, "row / feature sampling is not implemented");
  for (const char* k : {"lambda_l1", "max_delta_step", "path_smooth", "linear_lambda", "cegb_penalty_split", "monotone_penalty"})
    if (num(k, 0.0) > 0.0) bad(k, "not implemented");
  for (const char* k : {"extra_trees", "linear_tree", "use_nesterov_acc", "zero_as_missing", "is_unbalance", "use_quantized_grad"})
    if (flag(k)) bad(k, "not implemented");
  for (const char* k : {"monotone_constraints", "categorical_feature", "max_bin_by_feature", "interaction_constraints", "feature_contri",
                        "forcedsplits_filename", "forcedbins_filename", "cegb_penalty_feature_lazy", "cegb_penalty_feature_coupled"})
    if (nonempty_list(k)) bad(k, "not implemented");
  if (has("num_class") && std::stoi(kv.at("num_class")) != 1) bad("num_class", "single-output regression only");
  if (has("device_type") && kv.at("device_type") != "cuda" && kv.at("device_type") != "gpu" && kv.at("device_type") != "cpu")
    bad("device_type", "unknown device");
}

static const std::string* Find(const std::map<std::string, std::string>& kv, const std::string& k, std::initializer_list<const char*> al) {
  auto it = kv.find(k);
  if (it != kv.end()) return &it->second;
  for (const char* a : al) {
    it = kv.find(a);
    if (it != kv.end()) return &it->second;
  }
  return nullptr;
}
int Params::GetInt(const std::string& k, int d, std::initializer_list<const char*> al) const {
  const std::string* v = Find(kv, k, al);
  return v ? std::stoi(*v) : d;
}
double Params::GetDouble(const std::string& k, double d, std::initializer_list<const char*> al) const {
  const std::string* v = Find(kv, k, al);
  return v ? std::stod(*v) : d;
}
bool Params::GetBool(const std::string& k, bool d, std::initializer_list<const char*> al) const {
  const std::string* v = Find(kv, k, al);
  if (!v) return d;
  return *v == "true" || *v == "True" || *v == "1" || *v == "+";
}
std::string Params::GetString(const std::string& k, const std::string& d, std::initializer_list<const char*> al) const {
  const std::string* v = Find(kv, k, al);
  return v ? *v : d;
}

Dataset::Dataset(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, const Params& params)
    : num_data_(nrow), num_total_features_(ncol), params_(params) {
  if (data == nullptr || nrow <= 0 || ncol <= 0) Fatal("LGBM_DatasetCreateFromMat: empty data");
  if (data_type != 0 && data_type != 1) Fatal("Unknown data type in LGBM_DatasetCreateFromMat (float32 / float64 supported)");
  params.RejectUnsupported("Dataset");
  const int max_bin = params.GetInt("max_bin", 255);
  if (max_bin < 2 || max_bin > 255) Fatal("max_bin must be in [2, 255] for the CUDA tree learner (uint8 bins)");
  const int min_data_in_bin = params.GetInt("min_data_in_bin", 3);
  const int sample_cnt_cfg = params.GetInt("bin_construct_sample_cnt", 200000, {"subsample_for_bin"});
  const int data_random_seed = params.GetInt("data_random_seed", 1, {"data_seed"});
  const bool pre_filter = params.GetBool("feature_pre_filter", false);  // GPBoost default (include/LightGBM/config.h:649)
  const int min_data_in_leaf = params.GetInt("min_data_in_leaf", 20, {"min_data_per_leaf", "min_data", "min_child_samples"});
  auto at = [&](int64_t i, int j) {
    return data_type == 0 ? At<float>(data, nrow, ncol, is_row_major, i, j) : At<double>(data, nrow, ncol, is_row_major, i, j);
  };
  // ---- bin boundaries from a row sample, on the host (c_api.cpp:1182-1206 draws the rows; dataset_loader.cpp:600-700 one feature at a time)
  const std::vector<int> sample_rows = DrawSampleRows(nrow, std::min<int>(nrow, sample_cnt_cfg), data_random_seed);
  const int sample_cnt = (int)sample_rows.size();
  const int min_split_rows = static_cast<int>(static_cast<double>(min_data_in_leaf * (int64_t)sample_cnt) / nrow);  // dataset_loader.cpp:644
  bins_.resize(ncol);
#pragma omp parallel for schedule(dynamic)
  for (int j = 0; j < ncol; ++j) {
    std::vector<double> vals;
    vals.reserve(sample_cnt);
    for (int s = 0; s < sample_cnt; ++s) {
      const double v = at(sample_rows[s], j);
      if (std::fabs(v) > kZeroThreshold || std::isnan(v)) vals.push_back(v);  // zeros stay implicit
    }
    try {
      bins_[j] = BoundsFromSample(vals, (size_t)sample_cnt, max_bin, min_data_in_bin, min_split_rows, pre_filter);
    } catch (...) {
      bins_[j].num_bin = -1;  // re-raised below (no exceptions across the OpenMP region)
    }
  }
  for (int j = 0; j < ncol; ++j)
    if (bins_[j].num_bin < 0) Fatal("Missing values (NaN) in the feature matrix are not supported by the CUDA tree learner yet");
  for (int j = 0; j < ncol; ++j)
    if (!bins_[j].trivial) used_features_.push_back(j);
  BinOnDevice(data, data_type, nrow, ncol, is_row_major);
}

// Validation data (LGBM_DatasetCreateFromMat with a reference, c_api.cpp:1134-1160 -> DatasetLoader::ConstructFromSampleData with the
// reference's bin mappers): the training data's boundaries and feature set, so that the trees' bin thresholds apply to these rows
// (Dataset::CheckAlign, dataset.h). The values are binned on the device like the training data's.
Dataset::Dataset(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, const Params& params, const Dataset& reference)
    : num_data_(nrow), num_total_features_(ncol), params_(params) {
  if (data == nullptr || nrow <= 0 || ncol <= 0) Fatal("LGBM_DatasetCreateFromMat: empty data");
  if (data_type != 0 && data_type != 1) Fatal("Unknown data type in LGBM_DatasetCreateFromMat (float32 / float64 supported)");
  params.RejectUnsupported("Dataset");
  if (ncol != reference.num_total_features())
    Fatal("The number of features of the data (" + std::to_string(ncol) + ") differs from the reference Dataset's (" +
          std::to_string(reference.num_total_features()) + ")");
  for (int64_t i = 0; i < (int64_t)nrow * ncol; ++i) {
    const double v = data_type == 0 ? (double)static_cast<const float*>(data)[i] : static_cast<const double*>(data)[i];
    if (std::isnan(v)) Fatal("Missing values (NaN) in the feature matrix are not supported by the CUDA tree learner yet");
  }
  bins_ = reference.bins_;
  used_features_ = reference.used_features_;
  feature_names_ = reference.feature_names_;
  BinOnDevice(data, data_type, nrow, ncol, is_row_major);
}

bool Dataset::CheckAlign(const Dataset& other) const {  // Dataset::CheckAlign (include/LightGBM/dataset.h): same features, same bins
  if (num_total_features_ != other.num_total_features_ || used_features_ != other.used_features_) return false;
  for (int real : used_features_) {
    const FeatureBins &a = bins_[real], &b = other.bins_[real];
    if (a.num_bin != b.num_bin || a.upper_bounds != b.upper_bounds) return false;
  }
  return true;
}

void Dataset::BinOnDevice(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major) {
  // ---- value -> bin for every row: on the device, straight into the learner's row-major layout (csrc/dev/binning.cu)
  const int F = (int)used_features_.size();
  if (F == 0) return;
  fpad_ = (F + 31) / 32 * 32;
  device_ = GetRuntime().device;
  std::vector<int32_t> real(F), nb(F);
  std::vector<double> ub((size_t)F * 256, std::numeric_limits<double>::infinity());
  for (int k = 0; k < F; ++k) {
    const FeatureBins& fb = bins_[used_features_[k]];
    real[k] = used_features_[k];
    nb[k] = fb.num_bin;
    std::copy(fb.upper_bounds.begin(), fb.upper_bounds.end(), ub.begin() + (size_t)k * 256);
  }
  if (gpbdev_bin_matrix(device_, data, data_type, nrow, ncol, is_row_major, F, real.data(), nb.data(), ub.data(), 256, fpad_, &bins_dev_) != 0) {
    const std::string msg = gpbdev_bin_last_error();
    // Without a device the Dataset keeps its metadata (labels, names, boundaries) so that callers reach the error where the
    // reference's packages expect it — at Booster creation; there is no host binning path.
    if (msg.find("no CUDA device") != std::string::npos) { bins_dev_ = nullptr; bins_error_ = msg; }
    else Fatal(msg);
  }
}

Dataset::~Dataset() {
  if (bins_dev_ != nullptr) gpbdev_bin_free(device_, bins_dev_);
}

const uint8_t* Dataset::bins_device() const {
  if (bins_dev_ == nullptr) Fatal(bins_error_.empty() ? std::string("The Dataset holds no binned features") : bins_error_);
  return bins_dev_;
}

std::vector<uint8_t> Dataset::DownloadBins() const {
  std::vector<uint8_t> out((size_t)num_data_ * fpad_);
  if (gpbdev_bin_download(device_, bins_device(), num_data_, fpad_, out.data()) != 0) Fatal(gpbdev_bin_last_error());
  return out;
}

void Dataset::SetLabel(const float* label, int n) {
  if (n != num_data_) Fatal("Length of label is not same with #data");
  label_.assign(label, label + n);
}

std::vector<std::string> Dataset::feature_infos() const {
  std::vector<std::string> out;
  for (int j = 0; j < num_total_features_; ++j) {
    const FeatureBins& fb = bins_[j];
    if (fb.trivial) { out.push_back("none"); continue; }
    char buf[96];
    std::snprintf(buf, sizeof(buf), "[%.17g:%.17g]", fb.min_val, fb.max_val);
    out.push_back(buf);
  }
  return out;
}

}  // namespace gpb200
