// Request inputs -> the packed request row. A single-input model takes one tensor whose rows are in_dim values each, as
// always. A multi-input model (signature.inputs, e.g. BERT's input_ids / input_mask / segment_ids) takes one int32 tensor
// per declared input, [B, S] (or [S] for one row; a seed [B, 1] or [1]: input_width), and its request row is the
// concatenation of the inputs' rows in byte-wise sorted NAME order. The order depends on the names only, so the ingress rank of a forward hop packs a request
// without the owner's manifest; the owner checks the layout against its manifest (check_layout) before anything runs.
#pragma once
#include <string>
#include <vector>

#include "model.h"

namespace tfsc {

// a named request tensor as a front-end sees it (C ABI tensor, gRPC TensorProto view, REST column)
struct InTensor {
  std::string name;  // "" = unnamed: only a single tensor may omit its name
  int dtype = TFSC_DT_FLOAT;
  const void* data = nullptr;
  std::vector<int64_t> shape;
  int64_t n = 0;  // elements
};

// how a request is packed: its tensors in sorted name order and the values each contributes per row
struct InputLayout {
  std::vector<std::string> names;
  std::vector<int64_t> row_elems;
  int64_t n_elems = 0;  // all tensors
  int64_t rows = 0;     // several tensors: their common leading dimension (1 for rank-1 tensors); one tensor: 0 (from the model)
  int dtype = TFSC_DT_FLOAT;
  std::string error;    // a manifest-free check failed; reported after the model is resident, as every input error
  bool multi() const { return names.size() > 1; }
};

// Sorts `ts` by name and describes their packing. Several tensors must be named, distinct, int32 and share their batch
// dimension; a violation is recorded in layout.error (nothing is rejected before residency is ensured).
InputLayout layout_inputs(std::vector<InTensor>* ts);

// The owner's check of a layout against the model: for a multi-input model the names must be exactly the declared ones
// and every row its input's width values (S, 1 for a seed); a single-input model takes one tensor. Messages list the
// expected input names.
bool check_layout(const ModelDesc& d, const InputLayout& l, std::string* err);

// "'input_ids', 'input_mask', 'segment_ids'" (or the single input's name)
std::string expected_inputs(const ModelDesc& d);

// Writes `rows` packed rows to dst: row r is ts[0] row r | ts[1] row r | ... (one tensor: one memcpy of n values).
void pack_rows(const std::vector<InTensor>& ts, const InputLayout& l, int64_t rows, void* dst);

}  // namespace tfsc
