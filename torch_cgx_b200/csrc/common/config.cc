#include "config.h"

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

#include "quant_math.h"

namespace cgx {

int64_t env_int(const char* name, int64_t dflt) {
  const char* v = std::getenv(name);
  if (!v || !*v) return dflt;
  char* end = nullptr;
  long long r = std::strtoll(v, &end, 10);
  if (end == v) return dflt;
  return (int64_t)r;
}

double env_float(const char* name, double dflt) {
  const char* v = std::getenv(name);
  if (!v || !*v) return dflt;
  char* end = nullptr;
  double r = std::strtod(v, &end);
  if (end == v) return dflt;
  return r;
}

bool env_bool(const char* name, bool dflt) {
  const char* v = std::getenv(name);
  if (!v || !*v) return dflt;
  std::string s(v);
  std::transform(s.begin(), s.end(), s.begin(), ::tolower);
  if (s == "1" || s == "true" || s == "yes" || s == "on") return true;
  if (s == "0" || s == "false" || s == "no" || s == "off") return false;
  return dflt;
}

std::string env_str(const char* name, const std::string& dflt) {
  const char* v = std::getenv(name);
  return (v && *v) ? std::string(v) : dflt;
}

CommType env_comm_type(const char* name, CommType dflt, CommType mpi_equiv) {
  std::string s = env_str(name, "");
  std::transform(s.begin(), s.end(), s.begin(), ::toupper);
  if (s.empty()) return dflt;
  if (s == "SHM" || s == "P2P" || s == "NVLINK") return CommType::kP2P;
  if (s == "NCCL") return CommType::kNCCL;
  if (s == "GLOO") return CommType::kGloo;
  if (s == "MPI") return mpi_equiv;
  log_msg(0, "cgx: unknown communicator type '%s' for %s, using default", s.c_str(), name);
  return dflt;
}

ReductionType env_reduction_type(const char* name, ReductionType dflt) {
  std::string s = env_str(name, "");
  std::transform(s.begin(), s.end(), s.begin(), ::toupper);
  if (s.empty()) return dflt;
  if (s == "SRA") return ReductionType::kSRA;
  if (s == "RING") return ReductionType::kRing;
  if (s == "ALLTOALL" || s == "ALL_TO_ALL") return ReductionType::kAllToAll;
  log_msg(0, "cgx: unknown reduction type '%s' for %s, using default", s.c_str(), name);
  return dflt;
}

const char* to_string(CommType t) {
  switch (t) {
    case CommType::kP2P: return "P2P";
    case CommType::kNCCL: return "NCCL";
    default: return "GLOO";
  }
}
const char* to_string(ReductionType t) {
  switch (t) {
    case ReductionType::kSRA: return "SRA";
    case ReductionType::kRing: return "RING";
    default: return "ALLTOALL";
  }
}

CompressionEnv CompressionEnv::read() {
  CompressionEnv c;
  c.bits = (int)env_int(kEnvBits, kDefaultBits);
  if (c.bits < 1 || c.bits > 8) c.bits = kDefaultBits;  // anything else == off, like the reference (bits<=8 check)
  c.bucket_size = (int)std::max<int64_t>(1, env_int(kEnvBucketSize, kDefaultBucketSize));
  c.skip_incomplete = env_bool(kEnvSkipIncomplete, false);
  c.stochastic = env_bool(kEnvStochastic, false);
  c.seed = (uint64_t)env_int(kEnvSeed, 0);
  c.codec = parse_wire_format(env_str(kEnvFormat, ""), kEnvFormat);
  return c;
}

int parse_wire_format(const std::string& name, const char* what) {
  if (name.empty() || name == "maxmin") return kMaxMin;
  if (name == "e4m3") return kE4M3;
  if (name == "e5m2") return kE5M2;
  if (name == "e4m3_pow2") return kE4M3Pow2;
  if (name == "e5m2_pow2") return kE5M2Pow2;
  if (name == "e4m3_sr") return kE4M3SR;
  if (name == "e5m2_sr") return kE5M2SR;
  throw std::invalid_argument(std::string("cgx: ") + what +
                              " must be \"maxmin\", \"e4m3\", \"e5m2\", \"e4m3_pow2\", \"e5m2_pow2\", \"e4m3_sr\" or "
                              "\"e5m2_sr\", got \"" +
                              name + "\"");
}

EngineConfig EngineConfig::read() {
  EngineConfig c;
  int64_t mb = env_int(kEnvFusionMb, kDefaultFusionMb);
  c.fusion_bytes = std::max<int64_t>(kMinFusionBytes, mb << 20);
  c.min_compress_elems = (int)std::max<int64_t>(kMinCompressElems, env_int(kEnvMinimalSize, 0));
  c.fake_ratio = env_float(kEnvFakeRatio, 1.0);
  if (!(c.fake_ratio > 0.0) || c.fake_ratio > 1.0) c.fake_ratio = 1.0;
  c.inner_comm = env_comm_type(kEnvInnerComm, CommType::kP2P, CommType::kNCCL);
  c.cross_comm = env_comm_type(kEnvCrossComm, CommType::kNCCL, CommType::kNCCL);
  c.inner_reduction = env_reduction_type(kEnvInnerReduction, ReductionType::kSRA);
  c.cross_reduction = env_reduction_type(kEnvCrossReduction, ReductionType::kRing);
  if (env_bool(kEnvAllToAllReduction, false)) c.inner_reduction = ReductionType::kAllToAll;
  c.intra_broadcast = env_bool(kEnvIntraBroadcast, true);
  c.intra_compress = env_bool(kEnvIntraCompress, true);
  c.dummy_compression = env_bool(kEnvDummyCompression, false);
  c.remote_buf = env_bool(kEnvRemoteBuf, true);
  c.lanes = (int)env_int(kEnvLanes, 0);
  c.timeout_ms = std::max<int64_t>(1, env_int(kEnvTimeoutMs, 120000));
  c.local_size = (int)env_int(kEnvLocalSize, 0);
  c.min_lane_elems = (uint32_t)std::max<int64_t>(8, env_int(kEnvMinLaneElems, 4096));
  c.overlap_lanes = (int)std::max<int64_t>(0, env_int(kEnvOverlapLanes, 64));
  c.oneshot_max_bytes = std::max<int64_t>(0, env_int(kEnvOneshotMaxBytes, 2 << 20));
  return c;
}

int log_level() {
  static int lvl = (int)env_int(kEnvLogLevel, 0);
  return lvl;
}

void log_msg(int level, const char* fmt, ...) {
  if (level > log_level()) return;
  va_list ap;
  va_start(ap, fmt);
  std::vfprintf(stderr, fmt, ap);
  std::fputc('\n', stderr);
  va_end(ap);
}

}  // namespace cgx
