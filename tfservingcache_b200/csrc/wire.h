// Protobuf wire codec for the messages on the Predict path (SURVEY.md row W), hand-rolled:
// zero-copy views into the request bytes (tensor_content / packed float_val point into the
// caller's buffer) and a response writer that leaves a hole for the executor to fill.
// Field numbers: proto/tensorflow/serving/predict.pb.go:30-43,98-100; model.pb.go:27-91;
// proto/tensorflow/core/framework/tensor.pb.go:25-68; tensor_shape.pb.go:38-96.
#pragma once
#include <string>
#include <vector>

#include "common.h"

namespace tfsc {

struct TensorView {
  std::string name;
  int dtype = 0;
  std::vector<int64_t> shape;
  const uint8_t* content = nullptr;  // tensor_content (field 4)
  size_t content_len = 0;
  const uint8_t* packed_f32 = nullptr;  // packed float_val (field 5, wire type 2)
  size_t packed_f32_len = 0;
  std::vector<float> loose_f32;  // unpacked float_val entries
  std::vector<int32_t> ints;     // int_val entries (packed or not), field 7
  // product of the dims, or -1 if a dim is negative or the product overflows / exceeds kMaxTensorElements
  // (a client-controlled shape must never size an allocation unchecked)
  static constexpr int64_t kMaxTensorElements = (int64_t)1 << 31;
  int64_t num_elements() const {
    int64_t n = 1;
    for (auto d : shape) {
      if (d < 0) return -1;
      if (d != 0 && n > kMaxTensorElements / d) return -1;
      n *= d;
    }
    return n;
  }
};

struct PredictRequestView {
  std::string model_name, signature_name;
  bool has_version = false;
  int64_t version = 0;
  std::vector<TensorView> inputs;
  std::vector<std::string> output_filter;
};

bool decode_predict_request(const void* data, size_t len, PredictRequestView* out, std::string* err);
// fp32 elements of a DT_FLOAT tensor; `scratch` is used when the data is not contiguous in the
// request (unpacked float_val, scalar broadcast).
bool tensor_f32(const TensorView& t, const float** data, int64_t* n, std::vector<float>* scratch, std::string* err);

// int32 elements of a DT_INT32 tensor (tensor_content or int_val)
bool tensor_i32(const TensorView& t, const int32_t** data, int64_t* n, std::vector<int32_t>* scratch, std::string* err);

// Serialized PredictResponse{outputs{name: TensorProto{DT_FLOAT, shape, float_val}}, model_spec}
// split around the float payload: prefix | n_floats*4 payload bytes | suffix.
void predict_response_frame(const std::string& model_name, int64_t version, const std::string& signature_name,
                            const std::string& output_name, const std::vector<int64_t>& shape, std::string* prefix,
                            std::string* suffix);

// One output of a multi-output response: fp32 values go in packed float_val (field 5), int64 in packed int64_val
// (field 10), int32 in packed int_val (field 7), as TF-Serving's AsProtoField writes them.
struct OutTensor {
  std::string name;
  int dtype = TFSC_DT_FLOAT;
  std::vector<int64_t> shape;
  const void* data = nullptr;
  int64_t n = 0;
};
// PredictResponse{outputs (in the given order), model_spec}
std::string encode_predict_response(const std::string& model_name, int64_t version, const std::string& signature_name,
                                    const std::vector<OutTensor>& outs);
// SessionRunResponse{tensor = [NamedTensorProto{name, t}], model_spec}
std::string encode_session_run_response(const std::string& model_name, int64_t version, const std::string& signature_name,
                                        const OutTensor& t);

// ---- Classify / Regress (tfservingproxy.go:173-198): ClassificationRequest / RegressionRequest{model_spec=1, input=2
// Input{example_list=1{examples=1}, example_list_with_context=2{examples=1, context=2}}}, tf.Example{features=1{feature=1
// map<string, Feature{bytes_list=1, float_list=2{value=1 packed}, int64_list=3}>}} (proto/tensorflow/serving/
// {classification,regression,input}.pb.go, proto/tensorflow/core/example/{example,feature}.pb.go)
struct ExampleView {
  std::vector<std::pair<std::string, std::vector<float>>> features;  // numeric features (int64 values converted)
  const std::vector<float>* find(const std::string& key) const {
    for (auto& f : features)
      if (f.first == key) return &f.second;
    return nullptr;
  }
};
struct ExampleRequestView {
  std::string model_name, signature_name;
  bool has_version = false;
  int64_t version = 0;
  std::vector<ExampleView> examples;  // context features (example_list_with_context) are merged into every example
};
bool decode_example_request(const void* data, size_t len, ExampleRequestView* out, std::string* err);
// ClassificationResponse{result=1{classifications=1[{classes=1[{label=1, score=2}]}]}, model_spec=2}: n examples x c scores
std::string encode_classification_response(const std::string& model_name, int64_t version, const std::string& signature,
                                           const float* scores, int64_t n, int64_t c);
// RegressionResponse{result=1{regressions=1[{value=1}]}, model_spec=2}
std::string encode_regression_response(const std::string& model_name, int64_t version, const std::string& signature,
                                       const float* values, int64_t n);

// ---- SessionRun (tfservingproxy.go:233-244): SessionRunRequest{model_spec=1, feed=2[NamedTensorProto{name=1, tensor=2}],
// fetch=3, target=4}; SessionRunResponse{tensor=1[NamedTensorProto], model_spec=3} (session_service.pb.go, named_tensor.pb.go)
struct SessionRunView {
  std::string model_name, signature_name;
  bool has_version = false;
  int64_t version = 0;
  std::vector<TensorView> feeds;        // TensorView.name = the fed tensor name ("x:0")
  std::vector<std::string> fetch, target;
};
bool decode_session_run_request(const void* data, size_t len, SessionRunView* out, std::string* err);
// response split around the float payload like predict_response_frame
void session_run_response_frame(const std::string& model_name, int64_t version, const std::string& signature_name,
                                const std::string& tensor_name, const std::vector<int64_t>& shape, std::string* prefix,
                                std::string* suffix);

}  // namespace tfsc
