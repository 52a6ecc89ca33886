// epp_config.cpp — loader for the EndpointPickerConfig YAML the reference emits.
//
// The reference's router role writes this document into the ConfigMap mounted at
// /config/config.yaml of the EPP container (/root/reference/pkg/router/epp.go:58-81,
// 125-129) — see GenerateEPPConfig and the five generators in
// /root/reference/pkg/router/strategy.go:27-165, plus verbatim passthrough of
// role.EndpointPickerConfig (strategy.go:29-31).  This file accepts exactly that
// schema:
//   apiVersion: inference.networking.x-k8s.io/v1alpha1
//   kind: EndpointPickerConfig
//   plugins:            [{type, name?, parameters?}]
//   schedulingProfiles: [{name, plugins: [{pluginRef, weight?}]}]
// and maps the plugin types of strategy.go:55-60,74-75,89-90,104-105,129-150 onto
// fi_epp_config.  It is a small indentation-based YAML subset reader (block maps,
// block sequences, flow sequences of scalars, quoted scalars, comments) — enough
// for this schema, deliberately not a general YAML implementation.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/fi_epp.h"

namespace {

struct Node {
  enum Kind { SCALAR, MAP, LIST } kind = SCALAR;
  std::string scalar;
  std::vector<std::pair<std::string, std::unique_ptr<Node>>> map;
  std::vector<std::unique_ptr<Node>> list;
  const Node* get(const char* key) const {
    for (auto& kv : map)
      if (kv.first == key) return kv.second.get();
    return nullptr;
  }
};

struct Line {
  int indent;
  std::string text;  // without indentation, comments and trailing spaces
  int lineno;
};

struct ParseError {
  std::string msg;
};

std::string strip(const std::string& s) {
  size_t a = 0, b = s.size();
  while (a < b && (s[a] == ' ' || s[a] == '\t' || s[a] == '\r')) ++a;
  while (b > a && (s[b - 1] == ' ' || s[b - 1] == '\t' || s[b - 1] == '\r')) --b;
  return s.substr(a, b - a);
}

// remove a trailing "# comment" that is outside quotes
std::string strip_comment(const std::string& s) {
  char q = 0;
  for (size_t i = 0; i < s.size(); ++i) {
    char c = s[i];
    if (q) {
      if (c == q) q = 0;
    } else if (c == '"' || c == '\'') {
      q = c;
    } else if (c == '#' && (i == 0 || s[i - 1] == ' ' || s[i - 1] == '\t')) {
      return s.substr(0, i);
    }
  }
  return s;
}

std::string unquote(const std::string& s) {
  if (s.size() >= 2 && ((s.front() == '"' && s.back() == '"') || (s.front() == '\'' && s.back() == '\'')))
    return s.substr(1, s.size() - 2);
  return s;
}

std::vector<Line> split_lines(const char* y, size_t len) {
  std::vector<Line> out;
  size_t i = 0;
  int no = 0;
  while (i <= len) {
    size_t j = i;
    while (j < len && y[j] != '\n') ++j;
    ++no;
    std::string raw(y + i, j - i);
    i = j + 1;
    std::string nc = strip_comment(raw);
    int ind = 0;
    while ((size_t)ind < nc.size() && nc[ind] == ' ') ++ind;
    std::string t = strip(nc);
    if (t.empty() || t == "---") continue;
    out.push_back(Line{ind, t, no});
    if (j >= len) break;
  }
  return out;
}

// split "key: value" at the first ':' followed by space/end, outside quotes
bool split_kv(const std::string& t, std::string* k, std::string* v) {
  char q = 0;
  for (size_t i = 0; i < t.size(); ++i) {
    char c = t[i];
    if (q) {
      if (c == q) q = 0;
    } else if (c == '"' || c == '\'') {
      q = c;
    } else if (c == ':' && (i + 1 == t.size() || t[i + 1] == ' ')) {
      *k = unquote(strip(t.substr(0, i)));
      *v = strip(t.substr(i + 1));
      return true;
    }
  }
  return false;
}

std::unique_ptr<Node> parse_flow_or_scalar(const std::string& v, int lineno) {
  auto n = std::make_unique<Node>();
  if (!v.empty() && v.front() == '[') {
    if (v.back() != ']') throw ParseError{"line " + std::to_string(lineno) + ": unterminated flow sequence"};
    n->kind = Node::LIST;
    std::string inner = v.substr(1, v.size() - 2);
    std::string cur;
    char q = 0;
    auto push = [&]() {
      std::string s = strip(cur);
      if (!s.empty()) {
        auto e = std::make_unique<Node>();
        e->scalar = unquote(s);
        n->list.push_back(std::move(e));
      }
      cur.clear();
    };
    for (char c : inner) {
      if (q) {
        cur.push_back(c);
        if (c == q) q = 0;
      } else if (c == '"' || c == '\'') {
        q = c;
        cur.push_back(c);
      } else if (c == ',') {
        push();
      } else {
        cur.push_back(c);
      }
    }
    push();
    return n;
  }
  if (!v.empty() && v.front() == '{') throw ParseError{"line " + std::to_string(lineno) + ": flow mappings are not supported"};
  n->scalar = unquote(v);
  return n;
}

std::unique_ptr<Node> parse_block(std::vector<Line>& L, size_t& i, int indent);

// parse the entries of a mapping whose keys sit at `indent`
std::unique_ptr<Node> parse_map(std::vector<Line>& L, size_t& i, int indent) {
  auto n = std::make_unique<Node>();
  n->kind = Node::MAP;
  while (i < L.size() && L[i].indent == indent && L[i].text.compare(0, 2, "- ") != 0 && L[i].text != "-") {
    std::string k, v;
    if (!split_kv(L[i].text, &k, &v))
      throw ParseError{"line " + std::to_string(L[i].lineno) + ": expected 'key: value'"};
    int lineno = L[i].lineno;
    ++i;
    if (!v.empty()) {
      n->map.emplace_back(k, parse_flow_or_scalar(v, lineno));
    } else if (i < L.size() && (L[i].indent > indent ||
                                (L[i].indent == indent && (L[i].text.compare(0, 2, "- ") == 0 || L[i].text == "-")))) {
      // nested block; YAML allows a sequence value at the same indentation as its key
      n->map.emplace_back(k, parse_block(L, i, L[i].indent));
    } else {
      n->map.emplace_back(k, std::make_unique<Node>());  // empty scalar
    }
  }
  return n;
}

std::unique_ptr<Node> parse_list(std::vector<Line>& L, size_t& i, int indent) {
  auto n = std::make_unique<Node>();
  n->kind = Node::LIST;
  while (i < L.size() && L[i].indent == indent && (L[i].text.compare(0, 2, "- ") == 0 || L[i].text == "-")) {
    std::string rest = L[i].text == "-" ? "" : strip(L[i].text.substr(2));
    int lineno = L[i].lineno;
    if (rest.empty()) {
      ++i;
      if (i < L.size() && L[i].indent > indent)
        n->list.push_back(parse_block(L, i, L[i].indent));
      else
        n->list.push_back(std::make_unique<Node>());
      continue;
    }
    std::string k, v;
    if (split_kv(rest, &k, &v)) {
      // "- key: value" opens a mapping whose keys are indented by indent + 2
      int child = indent + 2 + (int)(L[i].text.size() - 2 - strip(L[i].text.substr(2)).size());
      L[i].indent = child;
      L[i].text = rest;
      n->list.push_back(parse_map(L, i, child));
    } else {
      n->list.push_back(parse_flow_or_scalar(rest, lineno));
      ++i;
    }
  }
  return n;
}

std::unique_ptr<Node> parse_block(std::vector<Line>& L, size_t& i, int indent) {
  if (L[i].text.compare(0, 2, "- ") == 0 || L[i].text == "-") return parse_list(L, i, indent);
  return parse_map(L, i, indent);
}

bool to_i64(const std::string& s, long long* out) {
  if (s.empty()) return false;
  char* end = nullptr;
  long long v = std::strtoll(s.c_str(), &end, 10);
  if (!end || *end != '\0') return false;
  *out = v;
  return true;
}

bool to_f64(const std::string& s, double* out) {
  if (s.empty()) return false;
  char* end = nullptr;
  double v = std::strtod(s.c_str(), &end);
  if (!end || *end != '\0') return false;
  *out = v;
  return true;
}

struct Plugin {
  std::string type, name;
  const Node* params = nullptr;
};

long long param_int(const Plugin& p, const char* key, long long dflt, bool* present = nullptr) {
  if (present) *present = false;
  if (!p.params) return dflt;
  const Node* n = p.params->get(key);
  if (!n || n->kind != Node::SCALAR) return dflt;
  long long v;
  if (!to_i64(n->scalar, &v)) throw ParseError{"plugin " + p.name + ": parameter " + key + " is not an integer"};
  if (present) *present = true;
  return v;
}

void set_err(char* err, size_t err_len, const std::string& m) {
  if (!err || !err_len) return;
  std::snprintf(err, err_len, "%s", m.c_str());
}

}  // namespace

// role_mask bit of one (label, value) pair of a by-label filter; a new pair is appended to cfg.labels
static uint32_t label_bit(fi_epp_config& cfg, const std::string& label, const std::string& value, uint32_t& next_bit) {
  for (uint32_t i = 0; i < cfg.n_labels; ++i)
    if (label == cfg.labels[i].label && value == cfg.labels[i].value) return cfg.labels[i].bit;
  uint32_t bit = 0;
  if (label == "fusioninfer.io/component-type") {
    if (value == "worker") bit = FI_ROLE_WORKER;
    else if (value == "prefiller") bit = FI_ROLE_PREFILLER;
    else if (value == "decoder") bit = FI_ROLE_DECODER;
  }
  if (!bit) {
    if (next_bit == 0) throw ParseError{"by-label: more than 29 distinct (label, value) pairs"};
    bit = next_bit;
    next_bit <<= 1;  // 0 after bit 31
  }
  if (cfg.n_labels >= FI_EPP_MAX_LABELS) throw ParseError{"by-label: too many (label, value) pairs"};
  fi_label_bit& lb = cfg.labels[cfg.n_labels];
  if (label.size() >= sizeof(lb.label)) throw ParseError{"by-label: label too long: " + label};
  if (value.size() >= sizeof(lb.value)) throw ParseError{"by-label: value too long: " + value};
  std::snprintf(lb.label, sizeof(lb.label), "%s", label.c_str());
  std::snprintf(lb.value, sizeof(lb.value), "%s", value.c_str());
  lb.bit = bit;
  ++cfg.n_labels;
  return bit;
}

// maxNumOfEndpoints of a max-score-picker: how many endpoints upstream's picker returns, best first (default 1)
static uint32_t picker_max_endpoints(const Plugin& p) {
  const Node* n = p.params ? p.params->get("maxNumOfEndpoints") : nullptr;
  if (!n) return 1;
  long long v = 0;
  if (n->kind != Node::SCALAR || !to_i64(n->scalar, &v) || v < 1 || v > (long long)FI_EPP_MAX_RANKED)
    throw ParseError{"max-score-picker " + p.name + ": maxNumOfEndpoints must be an integer in [1, " +
                     std::to_string(FI_EPP_MAX_RANKED) + "]"};
  return (uint32_t)v;
}

// The loader behind fi_epp_config_from_yaml and fi_epp_config_picker_endpoints.  picker_endpoints != NULL: also
// read each profile's max-score-picker maxNumOfEndpoints into picker_endpoints[profile] (1 when absent), and reject
// a value that is not an integer in [1, FI_EPP_MAX_RANKED].  With NULL that parameter is not looked at, so
// fi_epp_config_from_yaml accepts every document it accepted before the ranked pick existed.
static int load_config(const char* yaml, size_t len, fi_epp_config* cfg, uint32_t* picker_endpoints, char* err, size_t err_len) {
  try {
    std::vector<Line> lines = split_lines(yaml, len);
    if (lines.empty()) throw ParseError{"empty document"};
    size_t i = 0;
    std::unique_ptr<Node> root = parse_block(lines, i, lines[0].indent);
    if (i != lines.size()) throw ParseError{"line " + std::to_string(lines[i].lineno) + ": unexpected indentation"};
    if (root->kind != Node::MAP) throw ParseError{"top level must be a mapping"};

    const Node* kind = root->get("kind");
    if (!kind || kind->scalar != "EndpointPickerConfig") throw ParseError{"kind must be EndpointPickerConfig"};
    const Node* api = root->get("apiVersion");
    if (!api || api->scalar.rfind("inference.networking.x-k8s.io/", 0) != 0)
      throw ParseError{"apiVersion must be inference.networking.x-k8s.io/v1alpha1"};

    const Node* pl = root->get("plugins");
    if (!pl || pl->kind != Node::LIST) throw ParseError{"plugins: must be a sequence"};
    std::vector<Plugin> plugins;
    for (auto& e : pl->list) {
      if (e->kind != Node::MAP) throw ParseError{"plugins: entries must be mappings"};
      Plugin p;
      const Node* t = e->get("type");
      if (!t || t->scalar.empty()) throw ParseError{"plugin without type"};
      p.type = t->scalar;
      const Node* nm = e->get("name");
      p.name = (nm && !nm->scalar.empty()) ? nm->scalar : p.type;
      const Node* pr = e->get("parameters");
      if (pr && pr->kind == Node::MAP) p.params = pr;
      for (auto& q : plugins)
        if (q.name == p.name) throw ParseError{"duplicate plugin name " + p.name};
      plugins.push_back(p);
    }
    auto find_plugin = [&](const std::string& name) -> const Plugin* {
      for (auto& q : plugins)
        if (q.name == name) return &q;
      return nullptr;
    };

    fi_epp_config out = *cfg;
    out.n_profiles = 0;
    out.pd_enabled = 0;
    out.pd_decode_profile = out.pd_prefill_profile = 0;
    out.pd_threshold = 0.0;
    std::memset(out.profiles, 0, sizeof(out.profiles));

    // plugin-level parameters
    for (auto& p : plugins) {
      if (p.type == "prefix-cache-scorer") {
        bool has = false;
        // the reference spells the block size both ways (strategy.go:57 vs :147)
        long long b = param_int(p, "blockSize", 0, &has);
        if (!has) b = param_int(p, "hashBlockSize", 0, &has);
        if (has) {
          if (b <= 0 || b > (1 << 20)) throw ParseError{"prefix-cache-scorer: block size out of range"};
          out.block_bytes = (uint32_t)b;
        }
        long long m = param_int(p, "maxPrefixBlocksToMatch", 0, &has);
        if (has) {
          if (m <= 0 || m > (long long)FI_EPP_MAX_BLOCKS)
            throw ParseError{"prefix-cache-scorer: maxPrefixBlocksToMatch out of range (1.." +
                             std::to_string(FI_EPP_MAX_BLOCKS) + ")"};
          out.max_blocks = (uint32_t)m;
        }
        long long c = param_int(p, "lruCapacityPerServer", 0, &has);
        if (has) {
          if (c < 0 || c > 0x7FFFFFFFLL) throw ParseError{"prefix-cache-scorer: lruCapacityPerServer out of range"};
          out.lru_capacity = (uint32_t)c;
        }
      } else if (p.type == "pd-profile-handler") {
        out.pd_enabled = 1;
        if (p.params) {
          const Node* th = p.params->get("threshold");
          if (th && th->kind == Node::SCALAR && !th->scalar.empty()) {
            double v;
            if (!to_f64(th->scalar, &v)) throw ParseError{"pd-profile-handler: threshold is not a number"};
            out.pd_threshold = v;
          }
        }
      } else if (p.type == "max-score-picker" || p.type == "prefill-header-handler" ||
                 p.type == "single-profile-handler" || p.type == "by-label" ||
                 p.type == "kv-cache-utilization-scorer" || p.type == "queue-scorer" ||
                 p.type == "lora-affinity-scorer") {
        // handled through the profiles (or needs no parameters)
      } else {
        throw ParseError{"unsupported plugin type " + p.type};
      }
    }

    const Node* sp = root->get("schedulingProfiles");
    if (!sp || sp->kind != Node::LIST || sp->list.empty()) throw ParseError{"schedulingProfiles: must be a non-empty sequence"};
    if (sp->list.size() > FI_EPP_MAX_PROFILES) throw ParseError{"too many scheduling profiles"};
    bool have_decode = false, have_prefill = false;
    uint32_t next_bit = FI_ROLE_FIRST_FREE;
    out.n_labels = 0;
    std::memset(out.labels, 0, sizeof(out.labels));
    for (auto& e : sp->list) {
      if (e->kind != Node::MAP) throw ParseError{"schedulingProfiles: entries must be mappings"};
      fi_profile& prof = out.profiles[out.n_profiles];
      const Node* nm = e->get("name");
      std::string name = nm ? nm->scalar : std::string();
      if (name.empty()) throw ParseError{"scheduling profile without name"};
      if (name.size() >= sizeof(prof.name)) throw ParseError{"profile name too long: " + name};
      std::snprintf(prof.name, sizeof(prof.name), "%s", name.c_str());
      const Node* pp = e->get("plugins");
      if (!pp || pp->kind != Node::LIST) throw ParseError{"profile " + name + ": plugins must be a sequence"};
      bool has_picker = false;
      for (auto& ref : pp->list) {
        if (ref->kind != Node::MAP) throw ParseError{"profile " + name + ": plugin entries must be mappings"};
        const Node* rn = ref->get("pluginRef");
        if (!rn || rn->scalar.empty()) throw ParseError{"profile " + name + ": entry without pluginRef"};
        const Plugin* p = find_plugin(rn->scalar);
        if (!p) throw ParseError{"profile " + name + ": unknown pluginRef " + rn->scalar};
        long long weight = 1;
        const Node* wn = ref->get("weight");
        if (wn && !wn->scalar.empty()) {
          if (!to_i64(wn->scalar, &weight) || weight < 0 || weight > 0x7FFFFFFFLL)
            throw ParseError{"profile " + name + ": bad weight for " + rn->scalar};
        }
        uint32_t kind_id = 0;
        if (p->type == "prefix-cache-scorer") kind_id = FI_SCORER_PREFIX;
        else if (p->type == "kv-cache-utilization-scorer") kind_id = FI_SCORER_KV_UTIL;
        else if (p->type == "queue-scorer") kind_id = FI_SCORER_QUEUE;
        else if (p->type == "lora-affinity-scorer") kind_id = FI_SCORER_LORA;
        if (kind_id) {
          if (prof.n_scorers >= FI_EPP_MAX_SCORERS) throw ParseError{"profile " + name + ": too many scorers"};
          prof.scorers[prof.n_scorers].kind = kind_id;
          prof.scorers[prof.n_scorers].weight = (int32_t)weight;
          ++prof.n_scorers;
        } else if (p->type == "max-score-picker") {
          if (picker_endpoints && !has_picker) picker_endpoints[out.n_profiles] = picker_max_endpoints(*p);
          has_picker = true;
        } else if (p->type == "by-label") {
          // strategy.go:135-144 shows the schema: `label` + `validValues`.  Every (label, value) pair stands for
          // one bit of the endpoints' role_mask: the component-type values keep their fixed bits, any other pair
          // gets the next free one, recorded in cfg->labels for the host.  Filters of a profile are ANDed.
          if (!p->params) throw ParseError{"by-label " + p->name + ": missing parameters"};
          const Node* lab = p->params->get("label");
          if (!lab || lab->scalar.empty()) throw ParseError{"by-label " + p->name + ": missing label"};
          const Node* vv = p->params->get("validValues");
          if (!vv || vv->kind != Node::LIST || vv->list.empty())
            throw ParseError{"by-label " + p->name + ": validValues must be a non-empty sequence"};
          uint32_t mask = 0;
          for (auto& val : vv->list) {
            if (val->scalar.empty()) throw ParseError{"by-label " + p->name + ": empty value"};
            mask |= label_bit(out, lab->scalar, val->scalar, next_bit);
          }
          if (prof.role_mask == 0 && prof.n_more_filters == 0) {
            prof.role_mask = mask;
          } else {
            if (prof.n_more_filters >= FI_EPP_MAX_FILTERS - 1) throw ParseError{"profile " + name + ": too many by-label filters"};
            prof.more_filters[prof.n_more_filters++] = mask;
          }
        } else {
          throw ParseError{"profile " + name + ": plugin " + p->name + " (" + p->type + ") cannot be used in a profile"};
        }
      }
      if (!has_picker) throw ParseError{"profile " + name + ": no picker (max-score-picker) referenced"};
      if (name == "decode") {
        have_decode = true;
        out.pd_decode_profile = out.n_profiles;
      } else if (name == "prefill") {
        have_prefill = true;
        out.pd_prefill_profile = out.n_profiles;
      }
      ++out.n_profiles;
    }
    if (out.pd_enabled && !(have_decode && have_prefill))
      throw ParseError{"pd-profile-handler requires profiles named 'prefill' and 'decode'"};
    *cfg = out;
    return FI_OK;
  } catch (const ParseError& e) {
    set_err(err, err_len, e.msg);
    return FI_ERR_CONFIG;
  } catch (const std::exception& e) {
    set_err(err, err_len, e.what());
    return FI_ERR_CONFIG;
  }
}

extern "C" int fi_epp_config_from_yaml(const char* yaml, size_t len, fi_epp_config* cfg, char* err, size_t err_len) {
  if (!yaml || !cfg) {
    set_err(err, err_len, "null argument");
    return FI_ERR_INVALID;
  }
  return load_config(yaml, len, cfg, nullptr, err, err_len);
}

extern "C" int fi_epp_config_picker_endpoints(const char* yaml, size_t len, uint32_t out[FI_EPP_MAX_PROFILES], char* err,
                                              size_t err_len) {
  if (!yaml || !out) {
    set_err(err, err_len, "null argument");
    return FI_ERR_INVALID;
  }
  uint32_t k[FI_EPP_MAX_PROFILES] = {};  // profiles the document does not have stay 0
  fi_epp_config scratch{};
  const int rc = load_config(yaml, len, &scratch, k, err, err_len);
  if (rc != FI_OK) return rc;
  std::memcpy(out, k, sizeof(k));
  return FI_OK;
}
