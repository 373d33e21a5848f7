#include "provider.h"
#include "savedmodel.h"

#include <dirent.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <thread>

#include "parse.h"

namespace tfsc {

static bool is_dir(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}

static bool list_dir_sorted(const std::string& dir, std::vector<std::string>* names) {
  DIR* d = opendir(dir.c_str());
  if (!d) return false;
  while (dirent* e = readdir(d)) {
    std::string n = e->d_name;
    if (n != "." && n != "..") names->push_back(n);
  }
  closedir(d);
  std::sort(names->begin(), names->end());  // ioutil.ReadDir sorts by filename
  return true;
}

bool DiskModelProvider::find_src_path(const std::string& model_dir, int64_t version, std::string* out, std::string* err) {
  std::vector<std::string> names;
  if (!list_dir_sorted(model_dir, &names)) {
    *err = "open " + model_dir + ": no such file or directory";
    return false;
  }
  std::string match;
  int n_matches = 0;
  for (auto& n : names) {
    int64_t v;
    if (parse_int64(n, &v) && v == version && is_dir(model_dir + "/" + n)) {
      ++n_matches;
      match = n;  // several matches: the last one wins (diskmodelprovider.go:55-66)
    }
  }
  if (n_matches == 0) {
    *err = "No matching model found";
    return false;
  }
  *out = model_dir + "/" + match;
  return true;
}

static int64_t tree_size(const std::string& path) {
  struct stat st;
  if (stat(path.c_str(), &st) != 0) return 0;
  if (!S_ISDIR(st.st_mode)) return st.st_size;
  std::vector<std::string> names;
  list_dir_sorted(path, &names);
  int64_t total = 0;
  for (auto& n : names) total += tree_size(path + "/" + n);
  return total;
}

// A model name is one path component below baseDir. The REST regex already forbids '/', the gRPC ModelSpec.name does
// not, and the files found are parsed by native code in this process: refuse anything that could leave baseDir.
static bool safe_model_name(const std::string& name, std::string* err) {
  if (name.empty() || name == "." || name == ".." || name.find('/') != std::string::npos ||
      name.find('\0') != std::string::npos) {
    *err = "No matching model found";  // same answer as a model that does not exist (diskmodelprovider.go:67)
    return false;
  }
  return true;
}

int64_t DiskModelProvider::model_size(const std::string& name, int64_t version, std::string* err) {
  std::string src;
  if (!safe_model_name(name, err)) return -1;
  if (!find_src_path(base_dir_ + "/" + name, version, &src, err)) return -1;
  return tree_size(src);  // fix of diskmodelprovider.go:76-82 (dir inode size): real bytes
}

static bool read_file(const std::string& path, std::string* out) {
  int fd = open(path.c_str(), O_RDONLY);
  if (fd < 0) return false;
  struct stat st;
  fstat(fd, &st);
  out->resize(st.st_size);
  size_t got = 0;
  while (got < out->size()) {
    ssize_t r = read(fd, &(*out)[got], out->size() - got);
    if (r <= 0) break;
    got += r;
  }
  close(fd);
  return got == out->size();
}

std::shared_ptr<HostModel> DiskModelProvider::load_model(const std::string& name, int64_t version,
                                                         const HostAllocFn& alloc, std::string* err) {
  std::string src;
  if (!safe_model_name(name, err)) return nullptr;
  if (!find_src_path(base_dir_ + "/" + name, version, &src, err)) return nullptr;
  std::string mtxt;
  Json mj;
  auto m = std::make_shared<HostModel>();
  m->id = {name, version};
  if (!read_file(src + "/tfsc_model.json", &mtxt)) {
    if (!savedmodel_present(src)) {
      *err = "model " + name + ": " + src + "/tfsc_model.json not readable (not a tfsc-b200 bundle)";
      return nullptr;
    }
    // a TensorFlow SavedModel directory as TF-Serving would load it: import graph + variables on the fly
    SavedModelBundle sb;
    std::string ierr;
    if (!savedmodel_import(src, &sb, &ierr)) {
      *err = "model " + name + ": SavedModel import failed: " + ierr;
      return nullptr;
    }
    if (!json_parse(sb.manifest_json, &mj, err) || !parse_manifest(mj, &m->desc, err)) return nullptr;
    m->bytes = m->desc.weights_bytes;
    if (sb.weights.size() < m->bytes) {
      *err = "model " + name + ": imported weights shorter than manifest weights_bytes";
      return nullptr;
    }
    m->data = alloc(m->bytes, &m->release);
    if (!m->data) {
      *err = "host allocation of " + std::to_string(m->bytes) + " bytes failed";
      return nullptr;
    }
    memcpy(m->data, sb.weights.data(), m->bytes);
    return m;
  }
  if (!json_parse(mtxt, &mj, err) || !parse_manifest(mj, &m->desc, err)) return nullptr;
  std::string wpath = src + "/weights.bin";
  int fd = open(wpath.c_str(), O_RDONLY);
  if (fd < 0) {
    *err = "open " + wpath + " failed";
    return nullptr;
  }
  struct stat st;
  fstat(fd, &st);
  if ((size_t)st.st_size < m->desc.weights_bytes) {
    close(fd);
    *err = wpath + " is shorter than manifest weights_bytes";
    return nullptr;
  }
  m->bytes = m->desc.weights_bytes;
  m->data = alloc(m->bytes, &m->release);
  if (!m->data) {
    close(fd);
    *err = "host allocation of " + std::to_string(m->bytes) + " bytes failed";
    return nullptr;
  }
  size_t got = 0;
  while (got < m->bytes) {  // straight into pinned memory: no bounce buffer
    ssize_t r = pread(fd, (char*)m->data + got, std::min<size_t>(m->bytes - got, 1u << 30), got);
    if (r <= 0) break;
    got += r;
  }
  close(fd);
  if (got != m->bytes) {
    *err = "short read of " + wpath;
    return nullptr;
  }
  return m;
}

bool DiskModelProvider::check() { return true; }  // diskmodelprovider.go:85-88

// ------------------------------------------------------------------------- synthetic ------
static inline uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}

void SyntheticModelProvider::fill(float* dst, uint32_t seed, uint32_t tensor_id, uint64_t n, float scale, int threads) {
  const uint32_t k = mix32(seed * 0x9E3779B9u + tensor_id * 0x85EBCA6Bu + 0x165667B1u);
  auto work = [=](uint64_t lo, uint64_t hi) {
    for (uint64_t j = lo; j < hi; ++j) {
      const uint32_t h = mix32((uint32_t)j + k);
      const float u = (float)(h >> 8) * (1.0f / 16777216.0f);
      dst[j] = (u * 2.0f - 1.0f) * scale;
    }
  };
  if (threads <= 1 || n < (1u << 20)) {
    work(0, n);
    return;
  }
  std::vector<std::thread> ts;
  uint64_t per = (n + threads - 1) / threads;
  for (int t = 0; t < threads; ++t) {
    uint64_t lo = t * per, hi = std::min<uint64_t>(n, lo + per);
    if (lo < hi) ts.emplace_back(work, lo, hi);
  }
  for (auto& t : ts) t.join();
}

SyntheticModelProvider::SyntheticModelProvider(const Json& cfg) {
  std::string tmpl = cfg.get_str("modelProvider.synthetic.template", "mlp");
  prefix_ = cfg.get_str("modelProvider.synthetic.namePrefix", "m");
  count_ = cfg.get_int("modelProvider.synthetic.count", 1000);
  seed_base_ = cfg.get_int("modelProvider.synthetic.seedBase", 1000);
  threads_ = (int)cfg.get_int("modelProvider.synthetic.threads", std::min(16u, std::max(1u, std::thread::hardware_concurrency())));
  if (tmpl == "manifest") {
    // any "tfsc-b200-v1" manifest (e.g. the ResNet-50 graph built by modelformat.resnet50_manifest()):
    // weights are synthesized per op, tensor id 2*i (kernel, uniform with variance 1/fan_in) and 2*i+1 (bias)
    std::string err;
    const Json* m = cfg.get("modelProvider.synthetic.manifest");
    if (!m || !parse_manifest(*m, &desc_, &err)) {
      bad_ = "modelProvider.synthetic.manifest: " + (m ? err : std::string("missing"));
    }
  } else if (tmpl == "affine") {
    desc_ = make_affine_desc();
    affine_a_ = cfg.get_num("modelProvider.synthetic.a", 0.5);
    affine_b_ = cfg.get_num("modelProvider.synthetic.b", 2.0);
  } else {
    std::vector<int> dims;
    if (const Json* d = cfg.get("modelProvider.synthetic.dims"))
      for (auto& v : d->arr) dims.push_back((int)v.integer());
    if (dims.size() < 2) dims = {9216, 9216, 9216, 9216};
    desc_ = make_mlp_desc(dims, {});
  }
}

bool SyntheticModelProvider::index_of(const std::string& name, int64_t* j) const {
  if (name.size() <= prefix_.size() || name.compare(0, prefix_.size(), prefix_) != 0) return false;
  std::string digits = name.substr(prefix_.size());
  for (char c : digits)
    if (c < '0' || c > '9') return false;
  if (!parse_int64(digits, j)) return false;
  return *j >= 0 && *j < count_;
}

int64_t SyntheticModelProvider::model_size(const std::string& name, int64_t version, std::string* err) {
  int64_t j;
  if (!bad_.empty()) {
    *err = bad_;
    return -1;
  }
  if (!index_of(name, &j) || version < 1) {
    *err = "No matching model found";
    return -1;
  }
  return (int64_t)desc_.weights_bytes;
}

std::shared_ptr<HostModel> SyntheticModelProvider::load_model(const std::string& name, int64_t version,
                                                              const HostAllocFn& alloc, std::string* err) {
  int64_t j;
  if (!index_of(name, &j) || version < 1) {
    *err = "No matching model found";
    return nullptr;
  }
  auto m = std::make_shared<HostModel>();
  m->id = {name, version};
  m->desc = desc_;
  m->bytes = desc_.weights_bytes;
  m->data = alloc(m->bytes, &m->release);
  if (!m->data) {
    *err = "host allocation of " + std::to_string(m->bytes) + " bytes failed";
    return nullptr;
  }
  const uint32_t seed = (uint32_t)(seed_base_ + j + 100003 * (version - 1));
  float* base = static_cast<float*>(m->data);
  if (desc_.tmpl == Template::Affine) {
    memset(m->data, 0, m->bytes);
    base[desc_.a_off / 4] = (float)affine_a_;
    base[desc_.b_off / 4] = (float)affine_b_;
    return m;
  }
  if (desc_.tmpl == Template::Graph) {
    memset(m->data, 0, m->bytes);
    for (size_t i = 0; i < desc_.ops.size(); ++i) {
      const GraphOp& o = desc_.ops[i];
      const uint32_t t0 = (uint32_t)(8 * i);  // tensor ids of op i: 8*i + {0 kernel/gamma, 1 bias/beta, 2 word, 3 pos, 4 type}
      switch (o.kind) {
        case OpKind::Conv:
        case OpKind::Dense:
        case OpKind::TokenScore:  // the vocabulary projection, a 1x1 conv
        case OpKind::DepthwiseConv: {  // depthwise: one kh x kw filter per channel, fan-in kh * kw, cout = c
          const bool dw = o.kind == OpKind::DepthwiseConv;
          const uint64_t fan_in = (uint64_t)o.kh * o.kw * (dw ? 1 : o.c);
          fill(base + o.w_off / 4, seed, t0, fan_in * (dw ? o.c : o.cout), (float)std::sqrt(3.0 / (double)fan_in), threads_);
          fill(base + o.b_off / 4, seed, t0 + 1, (uint64_t)o.cout, 0.1f, 1);
          break;
        }
        case OpKind::LayerNorm:
        case OpKind::Embed: {
          if (!o.norm) {  // word and position tables only
            fill(base + o.word_off / 4, seed, t0 + 2, (uint64_t)o.vocab * o.c, 0.05f, threads_);
            fill(base + o.pos_off / 4, seed, t0 + 3, (uint64_t)o.max_pos * o.c, 0.05f, 1);
            break;
          }
          float* g = base + o.w_off / 4;
          fill(g, seed, t0, (uint64_t)o.c, 0.1f, 1);
          for (int c = 0; c < o.c; ++c) g[c] += 1.0f;  // gamma = 1 + 0.1 u
          fill(base + o.b_off / 4, seed, t0 + 1, (uint64_t)o.c, 0.1f, 1);
          if (o.kind == OpKind::Embed) {
            fill(base + o.word_off / 4, seed, t0 + 2, (uint64_t)o.vocab * o.c, 0.05f, threads_);
            fill(base + o.pos_off / 4, seed, t0 + 3, (uint64_t)o.max_pos * o.c, 0.05f, 1);
            fill(base + o.type_off / 4, seed, t0 + 4, (uint64_t)2 * o.c, 0.05f, 1);
          }
          break;
        }
        case OpKind::WindowAttention:  // the relative-position bias stays zero
        case OpKind::MaxPool: case OpKind::AvgPool: case OpKind::Attention: case OpKind::MaskGather:
        case OpKind::ChannelScale: case OpKind::PatchMerge: case OpKind::LastToken:
          break;
      }
    }
    return m;
  }
  for (size_t l = 0; l < desc_.layers.size(); ++l) {
    const DenseLayer& L = desc_.layers[l];
    const float ws = (float)std::sqrt(3.0 / (double)L.in);
    fill(base + L.w_off / 4, seed, (uint32_t)(2 * l), (uint64_t)L.in * L.out, ws, threads_);
    fill(base + L.b_off / 4, seed, (uint32_t)(2 * l + 1), (uint64_t)L.out, 0.1f, 1);
    // zero the alignment padding so the blob is fully deterministic
    size_t wend = L.w_off + (size_t)L.in * L.out * 4;
    memset((char*)m->data + wend, 0, L.b_off - wend);
    size_t bend = L.b_off + (size_t)L.out * 4;
    size_t next = (l + 1 < desc_.layers.size()) ? desc_.layers[l + 1].w_off : desc_.weights_bytes;
    memset((char*)m->data + bend, 0, next - bend);
  }
  return m;
}

std::unique_ptr<ModelProvider> create_provider(const Json& cfg, std::string* err) {
  std::string type = cfg.get_str("modelProvider.type", "");
  if (type == "diskProvider") {
    // code reads modelProvider.diskProvider.baseDir (main.go:159); README says basePath: accept both
    std::string dir = cfg.get_str("modelProvider.diskProvider.baseDir", cfg.get_str("modelProvider.diskProvider.basePath", ""));
    if (dir.empty()) {
      *err = "modelProvider.diskProvider.baseDir is not set";
      return nullptr;
    }
    return std::make_unique<DiskModelProvider>(dir);
  }
  if (type == "synthetic") return std::make_unique<SyntheticModelProvider>(cfg);
  if (type == "s3Provider" || type == "azBlobProvider") {
    *err = "modelProvider.type '" + type + "' is out of scope of this build (no network object stores on the box)";
    return nullptr;
  }
  *err = "Unsupported modelProvider.type: '" + type + "'";
  return nullptr;
}

}  // namespace tfsc

extern "C" {
int tfsc_disk_find_version_dir(const char* base_dir, const char* model_name, int64_t version, char* buf, size_t cap) {
  if (!base_dir || !model_name) return tfsc::fail(TFSC_E_INVALID, "disk_find_version_dir: bad arguments");
  std::string out, err;
  if (!tfsc::safe_model_name(model_name, &err)) return tfsc::fail(TFSC_E_NOT_FOUND, "%s", err.c_str());
  if (!tfsc::DiskModelProvider::find_src_path(std::string(base_dir) + "/" + model_name, version, &out, &err))
    return tfsc::fail(TFSC_E_NOT_FOUND, "%s", err.c_str());
  return tfsc::copy_out(out, buf, cap);
}
int64_t tfsc_disk_model_size(const char* base_dir, const char* model_name, int64_t version) {
  if (!base_dir || !model_name) return tfsc::fail(TFSC_E_INVALID, "disk_model_size: bad arguments");
  tfsc::DiskModelProvider p(base_dir);
  std::string err;
  int64_t s = p.model_size(model_name, version, &err);
  if (s < 0) return tfsc::fail(TFSC_E_NOT_FOUND, "%s", err.c_str());
  return s;
}

int tfsc_savedmodel_convert(const char* version_dir, const char* out_dir) {
  if (!version_dir || !out_dir) return tfsc::fail(TFSC_E_INVALID, "savedmodel_convert: bad arguments");
  tfsc::SavedModelBundle sb;
  std::string err;
  if (!tfsc::savedmodel_present(version_dir)) return tfsc::fail(TFSC_E_NOT_FOUND, "%s/saved_model.pb not found", version_dir);
  if (!tfsc::savedmodel_import(version_dir, &sb, &err)) return tfsc::fail(TFSC_E_INVALID, "%s", err.c_str());
  auto put = [&](const std::string& path, const void* d, size_t n) {
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    bool ok = fwrite(d, 1, n, f) == n;
    return fclose(f) == 0 && ok;
  };
  mkdir(out_dir, 0755);  // an existing directory is fine
  if (!put(std::string(out_dir) + "/weights.bin", sb.weights.data(), sb.weights.size()) ||
      !put(std::string(out_dir) + "/tfsc_model.json", sb.manifest_json.data(), sb.manifest_json.size()))
    return tfsc::fail(TFSC_E_INTERNAL, "cannot write the bundle into %s", out_dir);
  return 0;
}
uint32_t tfsc_crc32c(const void* data, size_t len) { return tfsc::crc32c(data, len); }
}
