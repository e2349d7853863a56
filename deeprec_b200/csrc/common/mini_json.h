// Minimal JSON reader (objects, arrays, strings, numbers, bools, null) for ModelConfig / saved_model.json / serving_versions.json.
// Used by both serving runtimes (csrc/host/cpu_serving.cc, csrc/cuda/serving_runtime.cu) and the saved-model reader (saved_model.h).
#pragma once
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

namespace drjson {

struct JVal {
  enum T { NUL, NUM, STR, ARR, OBJ, BOOL } t = NUL;
  double num = 0; std::string str; std::vector<JVal> arr; std::vector<std::pair<std::string, JVal>> obj;
  const JVal* get(const std::string& k) const { for (auto& kv : obj) if (kv.first == k) return &kv.second; return nullptr; }
  double n(const std::string& k, double d) const { auto* v = get(k); return v && (v->t == NUM || v->t == BOOL) ? v->num : d; }
  std::string s(const std::string& k, const std::string& d) const { auto* v = get(k); return v && v->t == STR ? v->str : d; }
};

struct JParser {
  const char* p; const char* e; bool ok = true; int depth = 0;
  void ws() { while (p < e && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) ++p; }
  JVal parse() {
    ws(); JVal v;
    if (p >= e || ++depth > 64) { ok = false; return v; }
    struct Leave { int& d; ~Leave() { --d; } } leave{depth};
    if (*p == '{') {
      v.t = JVal::OBJ; ++p; ws();
      if (p < e && *p == '}') { ++p; return v; }
      while (ok) {
        ws(); JVal k = parse();
        if (k.t != JVal::STR) { ok = false; break; }
        ws(); if (p >= e || *p != ':') { ok = false; break; } ++p;
        v.obj.emplace_back(k.str, parse()); ws();
        if (p < e && *p == ',') { ++p; continue; }
        if (p < e && *p == '}') { ++p; break; }
        ok = false;
      }
      return v;
    }
    if (*p == '[') {
      v.t = JVal::ARR; ++p; ws();
      if (p < e && *p == ']') { ++p; return v; }
      while (ok) {
        v.arr.push_back(parse()); ws();
        if (p < e && *p == ',') { ++p; continue; }
        if (p < e && *p == ']') { ++p; break; }
        ok = false;
      }
      return v;
    }
    if (*p == '"') {
      v.t = JVal::STR; ++p;
      while (p < e && *p != '"') {
        if (*p == '\\' && p + 1 < e) { ++p; char c = *p; v.str.push_back(c == 'n' ? '\n' : c == 't' ? '\t' : c); }
        else v.str.push_back(*p);
        ++p;
      }
      if (p < e) ++p; else ok = false;
      return v;
    }
    if (e - p >= 4 && !strncmp(p, "true", 4)) { v.t = JVal::BOOL; v.num = 1; p += 4; return v; }
    if (e - p >= 5 && !strncmp(p, "false", 5)) { v.t = JVal::BOOL; v.num = 0; p += 5; return v; }
    if (e - p >= 4 && !strncmp(p, "null", 4)) { p += 4; return v; }
    char* end = nullptr; v.num = strtod(p, &end);
    if (end == p || end > e) { ok = false; return v; }
    v.t = JVal::NUM; p = end; return v;
  }
};

inline bool ParseJson(const std::string& s, JVal* out) { JParser ps{s.c_str(), s.c_str() + s.size()}; *out = ps.parse(); return ps.ok; }

inline bool ReadFile(const std::string& path, std::string* out) {
  FILE* f = fopen(path.c_str(), "rb"); if (!f) return false;
  char buf[65536]; size_t n; out->clear();
  while ((n = fread(buf, 1, sizeof(buf), f)) > 0) out->append(buf, n);
  fclose(f); return true;
}

}  // namespace drjson
