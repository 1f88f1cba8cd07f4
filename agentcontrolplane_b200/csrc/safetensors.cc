// safetensors.cc — see safetensors.h.
#include "safetensors.h"

#include <fcntl.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <set>

namespace acp {

namespace {

bool read_text(const std::string& file, std::string* out) {
  FILE* f = fopen(file.c_str(), "rb");
  if (!f) return false;
  char buf[1 << 16];
  size_t n;
  out->clear();
  while ((n = fread(buf, 1, sizeof buf, f)) > 0) out->append(buf, n);
  fclose(f);
  return true;
}

bool is_dir(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}
bool is_file(const std::string& p) {
  struct stat st;
  return stat(p.c_str(), &st) == 0 && S_ISREG(st.st_mode);
}

size_t dtype_size(const std::string& d) {
  if (d == "BF16" || d == "F16") return 2;
  if (d == "F32") return 4;
  if (d == "F8_E4M3") return 1;   // FP8 codes (compressed-tensors float-quantized), used verbatim
  return 0;
}

}  // namespace

Checkpoint::~Checkpoint() {
  for (auto& m : maps_)
    if (m.base) munmap(m.base, m.len);
}

bool Checkpoint::map_file(const std::string& file, std::string* err) {
  const int fd = ::open(file.c_str(), O_RDONLY);
  if (fd < 0) { *err = "cannot open " + file; return false; }
  struct stat st;
  if (fstat(fd, &st) != 0 || st.st_size < 8) { close(fd); *err = file + ": not a safetensors file (too short)"; return false; }
  const size_t len = (size_t)st.st_size;
  void* base = mmap(nullptr, len, PROT_READ, MAP_PRIVATE, fd, 0);
  close(fd);
  if (base == MAP_FAILED) { *err = "mmap failed for " + file; return false; }
  maps_.push_back({base, len});
  const uint8_t* p = (const uint8_t*)base;
  uint64_t hlen = 0;
  for (int i = 7; i >= 0; --i) hlen = (hlen << 8) | p[i];
  if (hlen < 2 || hlen > len - 8 || hlen > (1ull << 30)) { *err = file + ": bad safetensors header length"; return false; }
  Json hdr;
  std::string perr;
  if (!Json::parse(std::string((const char*)p + 8, (size_t)hlen), &hdr, &perr) || !hdr.is_object()) {
    *err = file + ": safetensors header is not JSON (" + perr + ")";
    return false;
  }
  const uint8_t* buf = p + 8 + hlen;
  const size_t buf_len = len - 8 - (size_t)hlen;
  for (const auto& kv : hdr.members()) {
    if (kv.first == "__metadata__") continue;
    const Json& e = kv.second;
    StTensor t;
    t.dtype = e.get("dtype").as_string();
    for (const Json& d : e.get("shape").items()) t.shape.push_back(d.as_int());
    const Json& off = e.get("data_offsets");
    if (off.size() != 2) { *err = file + ": tensor " + kv.first + " has no data_offsets"; return false; }
    const long long b = off.items()[0].as_int(-1), en = off.items()[1].as_int(-1);
    if (b < 0 || en < b || (size_t)en > buf_len) { *err = file + ": tensor " + kv.first + " lies outside the file"; return false; }
    t.data = buf + b;
    t.nbytes = (size_t)(en - b);
    const size_t es = dtype_size(t.dtype);
    if (es != 0 && (size_t)t.numel() * es != t.nbytes) { *err = file + ": tensor " + kv.first + " size does not match its shape"; return false; }
    if (tensors_.count(kv.first)) { *err = "tensor " + kv.first + " appears in more than one file"; return false; }
    tensors_[kv.first] = std::move(t);
  }
  return true;
}

bool Checkpoint::open(const std::string& path, std::string* err) {
  std::string e;
  if (!err) err = &e;
  std::vector<std::string> files;
  if (is_dir(path)) {
    dir_ = path;
    std::string idx;
    if (read_text(path + "/model.safetensors.index.json", &idx)) {
      Json j;
      std::string perr;
      if (!Json::parse(idx, &j, &perr)) { *err = "model.safetensors.index.json: " + perr; return false; }
      std::set<std::string> seen;
      for (const auto& kv : j.get("weight_map").members())
        if (seen.insert(kv.second.as_string()).second) files.push_back(path + "/" + kv.second.as_string());
      if (files.empty()) { *err = "model.safetensors.index.json has an empty weight_map"; return false; }
    } else if (is_file(path + "/model.safetensors")) {
      files.push_back(path + "/model.safetensors");
    } else {
      *err = "no model.safetensors(.index.json) in " + path;
      return false;
    }
  } else if (is_file(path)) {
    const size_t slash = path.rfind('/');
    dir_ = slash == std::string::npos ? "." : path.substr(0, slash);
    files.push_back(path);
  } else {
    *err = "weights path does not exist: " + path;
    return false;
  }
  for (const std::string& f : files)
    if (!map_file(f, err)) return false;
  std::string cfg;
  if (read_text(dir_ + "/config.json", &cfg)) {
    std::string perr;
    if (!Json::parse(cfg, &config_, &perr) || !config_.is_object()) { *err = "config.json: " + perr; return false; }
    has_config_ = true;
  }
  return true;
}

const StTensor* Checkpoint::find(const std::string& name) const {
  auto it = tensors_.find(name);
  return it == tensors_.end() ? nullptr : &it->second;
}

std::string Checkpoint::index_json() const {
  Json out = Json::object();
  out.set("dir", Json(dir_));
  out.set("config", has_config_ ? config_ : Json());
  Json ts = Json::object();
  for (const auto& kv : tensors_) {
    Json t = Json::object();
    t.set("dtype", Json(kv.second.dtype));
    Json sh = Json::array();
    for (int64_t d : kv.second.shape) sh.push(Json((long long)d));
    t.set("shape", sh);
    t.set("nbytes", Json((long long)kv.second.nbytes));
    ts.set(kv.first, t);
  }
  out.set("tensors", ts);
  return out.dump();
}

bool st_to_bf16(const StTensor& t, size_t elem0, size_t n, uint16_t* out) {
  if (t.dtype == "BF16") {
    memcpy(out, t.data + elem0 * 2, n * 2);
    return true;
  }
  auto f32_to_bf16 = [](uint32_t u) -> uint16_t {
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40);  // quiet NaN
    return (uint16_t)((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);                 // round to nearest even
  };
  if (t.dtype == "F32") {
    const uint8_t* p = t.data + elem0 * 4;
    for (size_t i = 0; i < n; ++i) {
      uint32_t u;
      memcpy(&u, p + i * 4, 4);
      out[i] = f32_to_bf16(u);
    }
    return true;
  }
  if (t.dtype == "F16") {
    const uint8_t* p = t.data + elem0 * 2;
    for (size_t i = 0; i < n; ++i) {
      uint16_t h;
      memcpy(&h, p + i * 2, 2);
      const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
      uint32_t exp = (h >> 10) & 0x1f, man = h & 0x3ffu, u;
      if (exp == 0) {
        if (man == 0) u = sign;
        else {  // subnormal half -> normal float
          int e = -1;
          do { ++e; man <<= 1; } while (!(man & 0x400u));
          u = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ffu) << 13);
        }
      } else if (exp == 31) {
        u = sign | 0x7f800000u | (man << 13);
      } else {
        u = sign | ((exp + 112) << 23) | (man << 13);
      }
      out[i] = f32_to_bf16(u);
    }
    return true;
  }
  return false;
}

}  // namespace acp
