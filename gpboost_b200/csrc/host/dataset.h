// Dataset of this build: parameter parsing and bin-boundary finding on the host (sample-based, once per data set), value -> bin
// for every row on the device (csrc/dev/binning.cu, SURVEY §8 f3); owns the row-major uint8 bin matrix in HBM that the tree
// learner reads in place.
//
// Restates, for numerical features without missing values:
//   LGBM_DatasetCreateFromMat / ...Mats           src/LightGBM/c_api.cpp:1112-1232 (row sampling with Random(data_random_seed))
//   DatasetLoader::ConstructFromSampleData        src/LightGBM/io/dataset_loader.cpp:600-700 (filter_cnt, FindBin per column)
//   BinMapper::FindBin                            src/LightGBM/io/bin.cpp:325-520
//   FindBinWithZeroAsOneBin / GreedyFindBin       bin.cpp:241-311 / :78-155
//   NeedFilter                                    bin.cpp:53-75
//   BinMapper::ValueToBin                         include/LightGBM/bin.h:465-503
//   Random::Sample / NextFloat / NextInt          include/LightGBM/utils/random.h:41-109
// The boundary search is formulated on runs of the sorted sample (dataset.cpp); its outputs are pinned to the reference's bins by
// tests/test_binning_gpu.py (bins dumped by the reference's LGBM_DatasetDumpText).
#ifndef GPB200_DATASET_H_
#define GPB200_DATASET_H_
#include <cstdint>
#include <map>
#include <string>
#include <vector>

namespace gpb200 {

// key=value parameters ("parameters" strings of the LGBM_* API; Config::Str2Map, src/LightGBM/io/config.cpp)
struct Params {
  std::map<std::string, std::string> kv;
  static Params Parse(const char* s);  // keys are stored under their canonical names (aliases resolved)
  void RejectUnsupported(const char* where) const;  // throws for result-changing parameters this build does not implement
  int GetInt(const std::string& k, int dflt, std::initializer_list<const char*> aliases = {}) const;
  double GetDouble(const std::string& k, double dflt, std::initializer_list<const char*> aliases = {}) const;
  bool GetBool(const std::string& k, bool dflt, std::initializer_list<const char*> aliases = {}) const;
  std::string GetString(const std::string& k, const std::string& dflt, std::initializer_list<const char*> aliases = {}) const;
};

struct FeatureBins {
  std::vector<double> upper_bounds;  // bin_upper_bound_
  int num_bin = 0;
  bool trivial = false;
  double min_val = 0., max_val = 0.;
};

class Dataset {
 public:
  // data: nrow x ncol, float32 or float64 (C_API_DTYPE_*), row- or column-major
  Dataset(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, const Params& params);
  // binned with the bin mappers (feature set, upper bounds) of `reference` (validation data: LGBM_DatasetCreateFromMat with a reference)
  Dataset(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, const Params& params, const Dataset& reference);
  ~Dataset();
  // same feature set and bin boundaries (Dataset::CheckAlign): the trees of one can be walked on the bins of the other
  bool CheckAlign(const Dataset& other) const;
  Dataset(const Dataset&) = delete;
  Dataset& operator=(const Dataset&) = delete;
  int32_t num_data() const { return num_data_; }
  int num_total_features() const { return num_total_features_; }
  int num_features() const { return (int)used_features_.size(); }   // non-trivial ("inner") features
  int real_feature_index(int inner) const { return used_features_[inner]; }
  const FeatureBins& feature(int inner) const { return bins_[used_features_[inner]]; }
  const FeatureBins& feature_by_real_index(int real) const { return bins_[real]; }
  // device matrix, row-major num_data() x bins_row_stride() uint8 (padding features 0); throws when the process has no device
  const uint8_t* bins_device() const;
  int bins_row_stride() const { return fpad_; }
  int bins_device_id() const { return device_; }
  std::vector<uint8_t> DownloadBins() const;  // test hook (GPB200_DatasetGetBins)
  void SetLabel(const float* label, int n);
  const std::vector<float>& label() const { return label_; }
  bool has_label() const { return !label_.empty(); }
  const Params& params() const { return params_; }
  // feature names (Dataset::set_feature_names / feature_names, include/LightGBM/dataset.h): default "Column_<i>"
  const std::vector<std::string>& feature_names() const { return feature_names_; }
  void set_feature_names(const std::vector<std::string>& names) { feature_names_ = names; }
  // "[min:max]" per feature, "none" for a trivial one (BinMapper::bin_info_string, include/LightGBM/bin.h:195-215)
  std::vector<std::string> feature_infos() const;

 private:
  void BinOnDevice(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major);
  int32_t num_data_ = 0;
  int num_total_features_ = 0;
  Params params_;
  std::vector<FeatureBins> bins_;      // per real feature
  std::vector<int> used_features_;     // inner -> real
  uint8_t* bins_dev_ = nullptr;        // owned, on device_
  int fpad_ = 0, device_ = 0;
  std::string bins_error_;             // why bins_dev_ is null (no device in this process)
  std::vector<float> label_;
  std::vector<std::string> feature_names_;
};

}  // namespace gpb200
#endif
