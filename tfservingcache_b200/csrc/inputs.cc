#include "inputs.h"

#include <algorithm>
#include <cstring>

namespace tfsc {

InputLayout layout_inputs(std::vector<InTensor>* ts) {
  InputLayout l;
  std::sort(ts->begin(), ts->end(), [](const InTensor& a, const InTensor& b) { return a.name < b.name; });
  for (auto& t : *ts) {
    l.names.push_back(t.name);
    l.n_elems += t.n;
  }
  l.dtype = ts->empty() ? TFSC_DT_FLOAT : ts->front().dtype;
  if (ts->size() == 1) {
    l.row_elems.push_back(0);  // one tensor: the model's in_dim splits it into rows (Node::prepare)
    return l;
  }
  for (size_t i = 0; i < ts->size(); ++i) {
    const InTensor& t = (*ts)[i];
    const int64_t rows = t.shape.size() <= 1 ? 1 : t.shape[0];
    if (l.error.empty()) {
      if (t.name.empty()) l.error = "every input of a multi-input request needs a name";
      else if (i && t.name == (*ts)[i - 1].name) l.error = "input '" + t.name + "' is given twice";
      else if (t.dtype != TFSC_DT_INT32) l.error = "input '" + t.name + "' must be DT_INT32";
      else if (t.shape.empty() || rows <= 0 || t.n % rows) l.error = "input '" + t.name + "' needs a [batch, seq] or [seq] shape";
      else if (i && rows != l.rows)
        l.error = "inputs '" + (*ts)[0].name + "' and '" + t.name + "' have different batch sizes (" + std::to_string(l.rows) +
                  " vs " + std::to_string(rows) + ")";
    }
    if (i == 0) l.rows = rows;
    l.row_elems.push_back(rows > 0 ? t.n / rows : 0);
  }
  return l;
}

std::string expected_inputs(const ModelDesc& d) {
  if (d.inputs.empty()) return "'" + d.input_name + "'";
  std::string s;
  for (size_t i = 0; i < d.inputs.size(); ++i) s += (i ? ", '" : "'") + d.inputs[i].name + "'";
  return s;
}

bool check_layout(const ModelDesc& d, const InputLayout& l, std::string* err) {
  // every input but a seed holds S values per row (input_width); a seed's [batch, 1] is named after the rest
  const ModelInput* tokens = nullptr;
  std::string seeds;
  for (auto& mi : d.inputs)
    if (mi.role == InputRole::Seed) seeds += ", '" + mi.name + "' DT_INT32 [batch, 1]";
    else tokens = &mi;
  auto bad = [&](const std::string& why) {
    *err = why + "; model expects input" + (d.inputs.size() > 1 ? "s " : " ") + expected_inputs(d) +
           (d.inputs.empty() ? "" : ", DT_INT32 [batch, " + std::to_string(tokens ? tokens->width : 0) + "] each" + seeds);
    return false;
  };
  if (!l.error.empty()) return bad(l.error);
  if (d.inputs.empty()) {
    if (l.multi()) return bad("the request names " + std::to_string(l.names.size()) + " inputs");
    return true;  // one tensor for one input: the single-input checks of Node::prepare and the front-ends apply
  }
  for (auto& mi : d.inputs)
    if (std::find(l.names.begin(), l.names.end(), mi.name) == l.names.end()) return bad("input '" + mi.name + "' is missing");
  for (auto& n : l.names) {
    bool known = false;
    for (auto& mi : d.inputs) known = known || mi.name == n;
    if (!known) return bad(n.empty() ? std::string("an unnamed input") : "input '" + n + "' is not in the model signature");
  }
  if (l.dtype != TFSC_DT_INT32) return bad("the inputs must be DT_INT32");
  for (size_t i = 0; i < l.names.size(); ++i)  // the names are the declared ones, both in sorted order
    if (l.row_elems[i] != d.inputs[i].width)
      return bad("input '" + l.names[i] + "' has " + std::to_string(l.row_elems[i]) + " values per row, not " +
                 std::to_string(d.inputs[i].width));
  if (l.rows <= 0) return bad("the request has no rows");
  return true;
}

void pack_rows(const std::vector<InTensor>& ts, const InputLayout& l, int64_t rows, void* dst) {
  if (ts.size() == 1) {
    memcpy(dst, ts[0].data, (size_t)ts[0].n * 4);
    return;
  }
  char* out = static_cast<char*>(dst);
  for (int64_t r = 0; r < rows; ++r)
    for (size_t i = 0; i < ts.size(); ++i) {
      const size_t b = (size_t)l.row_elems[i] * 4;
      memcpy(out, static_cast<const char*>(ts[i].data) + (size_t)r * b, b);
      out += b;
    }
}

}  // namespace tfsc
