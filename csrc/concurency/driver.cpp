#include "driver.hpp"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <fstream>
#include <functional>
#include <iomanip>
#include <iostream>
#include <limits>
#include <set>
#include <sstream>

namespace hpcp {
namespace con {

namespace {

constexpr size_t kElemSize = sizeof(float);
constexpr const char* kComputeLetters = "CAT";

std::string join(const std::vector<std::string>& v, const std::string& sep) {
  std::string s;
  for (size_t i = 0; i < v.size(); ++i) {
    if (i) s += sep;
    s += v[i];
  }
  return s;
}

bool starts_with(const std::string& s, const std::string& p) { return s.rfind(p, 0) == 0; }

long parse_long(const std::string& flag, const std::string& text) {
  try {
    size_t pos = 0;
    const long v = std::stol(text, &pos);
    if (pos != text.size()) throw std::invalid_argument(text);
    return v;
  } catch (const std::exception&) {
    throw UsageError("Invalid integer '" + text + "' for '" + flag + "'");
  }
}

double parse_double(const std::string& flag, const std::string& text) {
  try {
    size_t pos = 0;
    const double v = std::stod(text, &pos);
    if (pos != text.size()) throw std::invalid_argument(text);
    return v;
  } catch (const std::exception&) {
    throw UsageError("Invalid number '" + text + "' for '" + flag + "'");
  }
}

std::string mode_header(const std::string& mode, const std::vector<std::string>& commands) {
  std::string s = mode + " | ";
  for (const auto& c : commands) s += c + " ";
  return s;
}

std::string json_escape(const std::string& s) {
  std::string o;
  for (char c : s) {
    if (c == '"' || c == '\\') o += '\\';
    o += c;
  }
  return o;
}

}  // namespace

std::string strip_twos(const std::string& token) {
  std::string out;
  out.reserve(token.size());
  for (char c : token)
    if (c != '2') out += c;
  return out;
}

bool is_compute_command(const std::string& cmd) {
  return cmd.size() == 1 && std::string(kComputeLetters).find(cmd[0]) != std::string::npos;
}

std::string tuned_parameter_of(const std::string& cmd) {
  if (cmd == "C") return "tripcount_C";
  if (cmd == "T") return "tripcount_T";  // tensor-core tile loop: duration ~ passes over the tile
  return "globalsize_" + cmd;
}

std::string usage_text(const std::string& program, const Backend& backend) {
  std::ostringstream os;
  os << "Usage: " << program << " (" << join(backend.modes(), " | ") << " | serial)\n"
     << "          [--commands CMD [CMD ...]]...   one concurrency experiment per --commands group\n"
     << "          [--queues N] [--repetitions N] [--min_bandwidth GB/s]\n"
     << "          [--tripcount_C N] [--globalsize_<CMD> N] [--globalsize_default_memory N]\n"
     << "          [--enable_profiling] [--verbose] [--json FILE]\n"
     << "\n"
     << "Backend: " << backend.name() << "\n"
     << "\n"
     << "Commands (a '2' inside a token is ignored, so M2D == MD):\n"
     << "  C      compute: every work-item runs 64*tripcount_C dependent FMAs\n"
     << "  A      compute: stream triad a = b + s*c over globalsize_A elements\n"
     << "  T      compute: wgmma tensor-core tile loop (CUDA backend only)\n"
     << "  X2Y    copy globalsize_XY floats from memory X to memory Y, with\n"
     << "           M  pageable host memory (malloc)\n"
     << "           H  pinned host memory\n"
     << "           D  device memory\n"
     << "           S  managed (shared) memory\n"
     << "           P  memory of a peer GPU, reached over NVLink\n"
     << "         endpoints available here: " << backend.memory_letters() << "\n"
     << "\n"
     << "Options:\n"
     << "  --tripcount_C N              [-1] FMA blocks per work-item; -1 autotunes it so that\n"
     << "                               every command of the run lasts about the same time\n"
     << "  --globalsize_<CMD> N         [-1] work-items (C) / elements (A, copies); -1 autotunes\n"
     << "  --globalsize_default_memory N  [-1] copy size before autotuning; -1 = 1e9 bytes\n"
     << "  --queues N                   [-1] streams / threads; -1 = one per command for\n"
     << "                               in_order and host_threads, otherwise 1\n"
     << "  --repetitions N              [10] the minimum over N runs is reported\n"
     << "  --min_bandwidth F            [-1] fail the group if the concurrent run moves fewer\n"
     << "                               than F GBytes/s; -1 = no floor\n"
     << "  --enable_profiling           also time every command on the device (events)\n"
     << "  --json FILE                  append one JSON row per group to FILE\n";
  return os.str();
}

Options parse_arguments(const std::vector<std::string>& args, const Backend& backend,
                        const std::string& program) {
  Options opt;
  opt.program = program;
  opt.cli_params = {{"globalsize_C", -1}, {"tripcount_C", -1}, {"globalsize_default_memory", -1}};
  if (args.empty()) throw UsageError("");

  opt.mode = args[0];
  {
    auto modes = backend.modes();
    modes.push_back("serial");
    if (std::find(modes.begin(), modes.end(), opt.mode) == modes.end())
      throw UsageError("Need to specify: (" + join(modes, " | ") + ")");
  }

  const std::string mem_letters = backend.memory_letters();
  const std::string compute_letters = backend.compute_letters();
  std::vector<std::string> current;
  auto flush_group = [&] {
    if (!current.empty()) opt.groups.push_back(current);
    current.clear();
  };
  auto value_of = [&](size_t& i, const std::string& flag) -> const std::string& {
    if (i + 1 >= args.size()) throw UsageError("Need to specify a value for '" + flag + "'");
    return args[++i];
  };

  for (size_t i = 1; i < args.size(); ++i) {
    const std::string& a = args[i];
    if (a == "--enable_profiling") {
      opt.enable_profiling = true;
    } else if (a == "--verbose") {
      opt.verbose = true;
    } else if (a == "--queues") {
      opt.n_queues = static_cast<int>(parse_long(a, value_of(i, a)));
    } else if (a == "--repetitions") {
      opt.n_repetitions = static_cast<int>(parse_long(a, value_of(i, a)));
      if (opt.n_repetitions < 1) throw UsageError("'--repetitions' must be >= 1");
    } else if (a == "--min_bandwidth") {
      opt.min_bandwidth = parse_double(a, value_of(i, a));
    } else if (a == "--json") {
      opt.json_path = value_of(i, a);
    } else if (starts_with(a, "--tripcount_") || starts_with(a, "--globalsize_")) {
      const std::string key = strip_twos(a.substr(2));
      opt.cli_params[key] = parse_long(a, value_of(i, a));
    } else if (starts_with(a, "--commands")) {
      flush_group();
    } else if (starts_with(a, "-")) {
      throw UsageError("Unsupported option: '" + a + "'");
    } else {
      const std::string cmd = strip_twos(a);
      bool ok = !cmd.empty();
      if (ok && cmd.size() == 1) {
        ok = compute_letters.find(cmd[0]) != std::string::npos;
      } else if (ok && cmd.size() == 2) {
        for (char c : cmd) ok = ok && mem_letters.find(c) != std::string::npos;
        // Host-to-host copies never touch the device: not a GPU concurrency question.
        const bool host_a = cmd[0] == 'M' || cmd[0] == 'H';
        const bool host_b = cmd[1] == 'M' || cmd[1] == 'H';
        ok = ok && !(host_a && host_b);
      } else {
        ok = false;
      }
      if (!ok) throw UsageError("Unsupported value for COMMAND: " + a);
      current.push_back(cmd);
    }
  }
  flush_group();
  if (opt.groups.empty())
    throw UsageError("Need to specify --commands (e.g. C, M2D, D2M, H2D, D2H, D2P)");
  return opt;
}

Params resolve_parameters(const Options& opt) {
  std::map<std::string, long> cli = opt.cli_params;
  for (const auto& g : opt.groups)
    for (const auto& c : g) {
      cli.emplace("globalsize_" + c, -1);
      if (c == "T") cli.emplace("tripcount_T", -1);
    }

  auto default_of = [&](const std::string& key) -> size_t {
    if (key == "globalsize_C") return 1;
    if (key == "tripcount_C") return 40000;
    if (key == "globalsize_T") return 132;  // one tile loop (CTA) per SM
    if (key == "tripcount_T") return 20000; // passes over the 128x256x64 tile (4 wgmma per warpgroup each)
    if (starts_with(key, "globalsize_")) {
      const long dm = cli.at("globalsize_default_memory");
      if (dm != -1) return static_cast<size_t>(dm);
      return static_cast<size_t>(1e9) / kElemSize;  // ~1 GB per buffer
    }
    return 0;
  };
  Params p;
  for (const auto& [k, v] : cli) p[k] = v == -1 ? default_of(k) : static_cast<size_t>(v);
  return p;
}

bool autotune(const Options& opt, Backend& backend, Params& params, std::ostream& out) {
  std::set<std::string> uniq;
  for (const auto& g : opt.groups) uniq.insert(g.begin(), g.end());

  auto cli_value = [&](const std::string& key) {
    auto it = opt.cli_params.find(key);
    return it == opt.cli_params.end() ? -1L : it->second;
  };
  bool wanted = false;
  for (const auto& c : uniq) wanted = wanted || cli_value(tuned_parameter_of(c)) == -1;
  if (!wanted || uniq.size() == 1) return false;

  out << "# Performing Autotuning to Balance Commands Times" << std::endl;
  BenchRequest req;
  req.mode = "serial";
  req.commands.assign(uniq.begin(), uniq.end());
  req.params = params;
  req.enable_profiling = opt.enable_profiling;
  req.n_queues = opt.n_queues;
  req.n_repetitions = opt.n_repetitions;
  req.verbose = opt.verbose;
  const BenchResult base = backend.run(req);

  // Target duration: the fastest *copy* at its maximum size (copies cannot grow,
  // compute can); if the run has no copy, the fastest command.
  long target = std::numeric_limits<long>::max();
  for (size_t i = 0; i < req.commands.size(); ++i)
    if (!is_compute_command(req.commands[i])) target = std::min(target, base.per_command_us[i]);
  if (target == std::numeric_limits<long>::max())
    for (long t : base.per_command_us) target = std::min(target, t);
  target = std::max(target, 1L);

  for (size_t i = 0; i < req.commands.size(); ++i) {
    const std::string key = tuned_parameter_of(req.commands[i]);
    if (cli_value(key) != -1) continue;  // pinned by the user
    const double t = static_cast<double>(std::max(base.per_command_us[i], 1L));
    const double scaled = static_cast<double>(target) / t * static_cast<double>(params[key]);
    params[key] = std::max<size_t>(1, static_cast<size_t>(scaled));
  }
  return true;
}

unsigned long long bytes_moved(const std::vector<std::string>& commands, const Params& params,
                               size_t elem_size) {
  unsigned long long bytes = 0;
  for (const auto& c : commands) {
    if (is_compute_command(c)) continue;
    auto it = params.find("globalsize_" + c);
    if (it != params.end()) bytes += static_cast<unsigned long long>(it->second) * elem_size;
  }
  return bytes;
}

std::string time_with_bandwidth(long us, unsigned long long bytes) {
  std::ostringstream os;
  os << us << "us";
  if (bytes != 0) {
    const double bw = 1e-3 * static_cast<double>(bytes) / static_cast<double>(std::max(us, 1L));
    os << " (" << bw << " GBytes/s)";
  }
  return os.str();
}

Verdict judge(double max_speedup, double speedup, double gbytes_per_s, double min_bandwidth,
              unsigned long long bytes) {
  if (bytes != 0 && min_bandwidth >= 0 && gbytes_per_s < min_bandwidth)
    return Verdict::kBandwidthFloor;
  if (max_speedup >= (1.0 + kSpeedupTolerance) * speedup) return Verdict::kFarFromTheoretical;
  return Verdict::kSuccess;
}

std::string verdict_text(Verdict v) {
  switch (v) {
    case Verdict::kBandwidthFloor: return "FAILURE: Minimun Bandwish not reached";
    case Verdict::kFarFromTheoretical: return "FAILURE: Far from Theoretical Speedup";
    case Verdict::kSuccess: return "SUCCESS: Close from Theoretical Speedup";
  }
  return "";
}

std::string verdict_line(const std::string& mode, const std::vector<std::string>& commands,
                         Verdict v) {
  return "## " + mode_header(mode, commands) + "| " + verdict_text(v);
}

GroupReport run_group(const Options& opt, Backend& backend, const Params& params,
                      const std::vector<std::string>& commands, std::ostream& out,
                      std::ostream& err) {
  GroupReport rep;
  rep.commands = commands;
  out << "# " << mode_header(opt.mode, commands) << "| Starting Benchmarking..." << std::endl;

  BenchRequest req;
  req.commands = commands;
  req.params = params;
  req.enable_profiling = opt.enable_profiling;
  req.n_queues = opt.n_queues;
  req.n_repetitions = opt.n_repetitions;
  req.verbose = opt.verbose;

  // 1. serial reference
  req.mode = "serial";
  const BenchResult serial = backend.run(req);
  rep.serial_total_us = serial.total_us;
  rep.serial_command_us = serial.per_command_us;
  out << "Minimum Measured Total Time Serial: " << serial.total_us << "us" << std::endl;
  for (size_t i = 0; i < commands.size(); ++i) {
    out << "  Minimum Time Command " << i << " (" << std::setw(3) << commands[i] << "): "
        << time_with_bandwidth(serial.per_command_us[i], bytes_moved({commands[i]}, params, kElemSize));
    if (opt.enable_profiling && i < serial.device_us.size() && serial.device_us[i] >= 0)
      out << " [device " << serial.device_us[i] << "us]";
    out << std::endl;
  }
  const long slowest =
      std::max(1L, *std::max_element(serial.per_command_us.begin(), serial.per_command_us.end()));
  rep.max_speedup = static_cast<double>(serial.total_us) / static_cast<double>(slowest);
  out << "Maximum Theoretical Speedup: " << rep.max_speedup << "x" << std::endl;
  if (rep.max_speedup <= kUnbalanceWarning)
    err << "  WARNING: Large Unbalance Between Commands" << std::endl;

  // 2. concurrent run
  req.mode = opt.mode;
  const BenchResult conc = backend.run(req);
  rep.concurrent_total_us = conc.total_us;
  rep.device_total_us = conc.device_total_us;
  rep.bytes = bytes_moved(commands, params, kElemSize);
  rep.concurrent_gbytes_per_s =
      1e-3 * static_cast<double>(rep.bytes) / static_cast<double>(std::max(conc.total_us, 1L));
  out << "Minimum Measured Total Time //: " << time_with_bandwidth(conc.total_us, rep.bytes);
  if (opt.enable_profiling && conc.device_total_us >= 0)
    out << " [device " << conc.device_total_us << "us]";
  out << std::endl;
  rep.speedup =
      static_cast<double>(serial.total_us) / static_cast<double>(std::max(conc.total_us, 1L));
  out << "Speedup Relative to Serial: " << rep.speedup << "x" << std::endl;

  // 3. verdict
  rep.verdict = judge(rep.max_speedup, rep.speedup, rep.concurrent_gbytes_per_s,
                      opt.min_bandwidth, rep.bytes);
  out << verdict_line(opt.mode, commands, rep.verdict) << std::endl;
  return rep;
}

namespace {

void append_json_row(const std::string& path, const Options& opt, const Backend& backend,
                     const Params& params, const GroupReport& r) {
  std::ofstream f(path, std::ios::app);
  if (!f) return;
  f << "{\"pattern\":\"concurency\",\"backend\":\"" << json_escape(backend.name())
    << "\",\"mode\":\"" << json_escape(opt.mode) << "\",\"commands\":[";
  for (size_t i = 0; i < r.commands.size(); ++i)
    f << (i ? "," : "") << "\"" << json_escape(r.commands[i]) << "\"";
  f << "],\"serial_total_us\":" << r.serial_total_us << ",\"serial_command_us\":[";
  for (size_t i = 0; i < r.serial_command_us.size(); ++i)
    f << (i ? "," : "") << r.serial_command_us[i];
  f << "],\"concurrent_total_us\":" << r.concurrent_total_us
    << ",\"device_total_us\":" << r.device_total_us << ",\"max_speedup\":" << r.max_speedup
    << ",\"speedup\":" << r.speedup << ",\"bytes\":" << r.bytes
    << ",\"gbytes_per_s\":" << r.concurrent_gbytes_per_s << ",\"overlap_fraction\":";
  // overlap % = (serial - concurrent) / (serial - slowest): 1 = perfect overlap.
  const long slowest =
      *std::max_element(r.serial_command_us.begin(), r.serial_command_us.end());
  const double denom = static_cast<double>(r.serial_total_us - slowest);
  f << (denom > 0 ? static_cast<double>(r.serial_total_us - r.concurrent_total_us) / denom : 0.0);
  f << ",\"params\":{";
  bool first = true;
  for (const auto& c : r.commands) {
    const std::string k = tuned_parameter_of(c);
    auto it = params.find(k);
    if (it == params.end()) continue;
    f << (first ? "" : ",") << "\"" << k << "\":" << it->second;
    first = false;
  }
  f << "},\"verdict\":\"" << (r.verdict == Verdict::kSuccess ? "SUCCESS" : "FAILURE") << "\"}\n";
}

}  // namespace

int run(const std::vector<std::string>& argv_tail, Backend& backend, std::ostream& out,
        std::ostream& err, const std::string& program) {
  Options opt;
  try {
    opt = parse_arguments(argv_tail, backend, program);
  } catch (const UsageError& e) {
    if (std::string(e.what()).size()) out << "ERROR: " << e.what() << std::endl;
    out << usage_text(program, backend) << std::endl;
    return 1;
  }

  Params params = resolve_parameters(opt);
  autotune(opt, backend, params, out);

  std::set<std::string> uniq;
  for (const auto& g : opt.groups) uniq.insert(g.begin(), g.end());
  out << "Parameters used:" << std::endl;
  for (const auto& c : uniq) {
    const std::string key = tuned_parameter_of(c);
    out << "  " << key << ": " << params[key] << std::endl;
    if (c == "C") out << "  globalsize_C: " << params["globalsize_C"] << std::endl;
    if (c == "T") out << "  globalsize_T: " << params["globalsize_T"] << std::endl;
  }

  int status = 0;
  for (const auto& commands : opt.groups) {
    const GroupReport rep = run_group(opt, backend, params, commands, out, err);
    if (rep.verdict != Verdict::kSuccess) status = 1;
    if (!opt.json_path.empty()) append_json_row(opt.json_path, opt, backend, params, rep);
  }
  return status;
}

// --------------------------------------------------------------- FakeBackend ----
namespace {

class FakeBackend final : public Backend {
 public:
  explicit FakeBackend(const std::string& spec) {
    std::stringstream ss(spec);
    std::string item;
    while (std::getline(ss, item, ',')) {
      const auto eq = item.find('=');
      if (eq == std::string::npos) continue;
      const std::string k = item.substr(0, eq);
      const std::string text = item.substr(eq + 1);
      char* end = nullptr;
      const double v = std::strtod(text.c_str(), &end);  // strtod: subnormal values are values, not errors
      if (text.empty() || end == nullptr || *end != '\0')
        throw std::invalid_argument("fake backend: bad number in '" + item + "' (expected name=value,...)");
      if (k == "overlap")
        overlap_ = v;
      else
        coef_[k] = v;
    }
  }
  std::string name() const override { return "fake"; }
  std::vector<std::string> modes() const override {
    return {"in_order", "out_of_order", "host_threads", "nowait", "fused"};
  }
  std::string memory_letters() const override { return "MDHSP"; }
  std::string compute_letters() const override { return "CAT"; }

  BenchResult run(const BenchRequest& req) override {
    BenchResult r;
    double sum = 0, mx = 0;
    for (const auto& c : req.commands) {
      const double coef = coef_.count(c) ? coef_.at(c) : 1e-3;
      const double t = coef * static_cast<double>(require_param(req, tuned_parameter_of(c)));
      r.per_command_us.push_back(static_cast<long>(std::llround(t)));
      sum += t;
      mx = std::max(mx, t);
    }
    if (req.mode == "serial") {
      r.total_us = 0;
      for (long t : r.per_command_us) r.total_us += t;
    } else {
      r.total_us = static_cast<long>(std::llround(mx + (1.0 - overlap_) * (sum - mx)));
      r.per_command_us.clear();
    }
    return r;
  }

 private:
  std::map<std::string, double> coef_;
  double overlap_ = 1.0;
};

}  // namespace

std::unique_ptr<Backend> make_fake_backend(const std::string& spec) {
  return std::make_unique<FakeBackend>(spec);
}

}  // namespace con
}  // namespace hpcp
