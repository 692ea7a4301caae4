// Environment-variable configuration surface. Same names and defaults as the
// reference (/root/reference/src/common/common.h:24-41,
// /root/reference/src/common/utils.cc:25-91, README.md:80-88), plus a few
// implementation-specific knobs (CGX_LANES, CGX_TIMEOUT_MS, CGX_STOCHASTIC, CGX_SEED...).
//
// Like the reference, the *compression* parameters (bits, bucket size,
// skip-incomplete) are re-read on every allreduce so tests and tuners can flip
// them between calls (/root/reference/src/common/compressor.cc:39-45,258-263);
// the *structural* parameters (fusion size, transports, lanes) are read once
// when an engine is constructed.
#pragma once
#include <cstdint>
#include <string>

namespace cgx {

// names (kept byte-identical to the reference where they exist there)
constexpr const char* kEnvBits = "CGX_COMPRESSION_QUANTIZATION_BITS";
constexpr const char* kEnvBucketSize = "CGX_COMPRESSION_BUCKET_SIZE";
constexpr const char* kEnvSkipIncomplete = "CGX_COMPRESSION_SKIP_INCOMPLETE_BUCKETS";
constexpr const char* kEnvMinimalSize = "CGX_COMPRESSION_MINIMAL_SIZE";
constexpr const char* kEnvFakeRatio = "CGX_COMPRESSION_FAKE_RATIO";
constexpr const char* kEnvFusionMb = "CGX_FUSION_BUFFER_SIZE_MB";
constexpr const char* kEnvInnerComm = "CGX_INNER_COMMUNICATOR_TYPE";
constexpr const char* kEnvCrossComm = "CGX_CROSS_COMMUNICATOR_TYPE";
constexpr const char* kEnvInnerReduction = "CGX_INNER_REDUCTION_TYPE";
constexpr const char* kEnvCrossReduction = "CGX_CROSS_REDUCTION_TYPE";
constexpr const char* kEnvIntraBroadcast = "CGX_INTRA_BROADCAST";
constexpr const char* kEnvIntraCompress = "CGX_INTRA_COMPRESS";
constexpr const char* kEnvRemoteBuf = "CGX_REMOTE_BUF_COMPRESSION";
constexpr const char* kEnvDummyCompression = "CGX_DEBUG_DUMMY_COMPRESSION";
constexpr const char* kEnvAllToAllReduction = "CGX_DEBUG_ALL_TO_ALL_REDUCTION";
// new in this implementation
constexpr const char* kEnvStochastic = "CGX_STOCHASTIC_ROUNDING";  // runtime QSGD switch (ref: build flag QSGD_DETERMENISTIC)
constexpr const char* kEnvSeed = "CGX_SEED";
constexpr const char* kEnvLanes = "CGX_LANES";                      // CTAs of the fused kernel (0 = auto)
constexpr const char* kEnvTimeoutMs = "CGX_TIMEOUT_MS";             // device-side flag wait timeout
constexpr const char* kEnvLocalSize = "CGX_LOCAL_SIZE";             // ranks per node override (simulated multi-node)
constexpr const char* kEnvLogLevel = "CGX_LOG_LEVEL";               // 0 silent, 1 info, 2 debug
constexpr const char* kEnvMinLaneElems = "CGX_MIN_LANE_ELEMS";
constexpr const char* kEnvOneshotMaxBytes = "CGX_ONESHOT_MAX_BYTES";  // messages up to this size take the one-shot kernel (0 = never)
constexpr const char* kEnvOverlapLanes = "CGX_OVERLAP_LANES";  // CTAs of a DDP-bucket allreduce that overlaps with backward (0 = no cap)
constexpr const char* kEnvVmm = "CGX_VMM";                      // 0: cudaMalloc + cudaIpc heap instead of VMM + fd handles
constexpr const char* kEnvNvls = "CGX_NVLS";                    // 0: never create the NVLS multicast mapping
constexpr const char* kEnvNvlsReduce = "CGX_NVLS_REDUCE";       // 0: raw layers use the two-shot path even with NVLS
constexpr const char* kEnvFormat = "CGX_COMPRESSION_FORMAT";    // wire format of the allreduce's 8-bit layers:
                                                                // unset / "maxmin", "e4m3" or "e5m2"

constexpr int kDefaultBits = 32;          // 32 == compression off
constexpr int kDefaultBucketSize = 512;   // reference compressor.h:32
constexpr int kMinCompressElems = 16;     // reference compressor.cc:36
constexpr int kDefaultFusionMb = 64;      // reference common.h:40
constexpr int64_t kMinFusionBytes = 2048; // reference common.h:41

enum class CommType { kP2P, kNCCL, kGloo };      // reference: SHM / NCCL / MPI
enum class ReductionType { kSRA, kRing, kAllToAll };

int64_t env_int(const char* name, int64_t dflt);
double env_float(const char* name, double dflt);
bool env_bool(const char* name, bool dflt);
std::string env_str(const char* name, const std::string& dflt);
// "SHM" (reference default, host staged) maps to the P2P peer-memory path here;
// "MPI" has no equivalent on this stack and maps to `mpi_equiv`.
CommType env_comm_type(const char* name, CommType dflt, CommType mpi_equiv);
ReductionType env_reduction_type(const char* name, ReductionType dflt);
const char* to_string(CommType t);
const char* to_string(ReductionType t);

// Re-read on every allreduce.
struct CompressionEnv {
  int bits = kDefaultBits;
  int bucket_size = kDefaultBucketSize;
  bool skip_incomplete = false;
  bool stochastic = false;
  uint64_t seed = 0;
  int codec = 0;  // WireCodec (quant_math.h) of CGX_COMPRESSION_FORMAT; std::invalid_argument on an unknown name
  static CompressionEnv read();
};
// "maxmin" (or empty) / "e4m3" / "e5m2" -> WireCodec; std::invalid_argument naming `what` otherwise
int parse_wire_format(const std::string& name, const char* what);

// Read once per engine.
struct EngineConfig {
  int64_t fusion_bytes = (int64_t)kDefaultFusionMb << 20;
  int min_compress_elems = kMinCompressElems;
  double fake_ratio = 1.0;
  CommType inner_comm = CommType::kP2P;
  CommType cross_comm = CommType::kNCCL;
  ReductionType inner_reduction = ReductionType::kSRA;
  ReductionType cross_reduction = ReductionType::kRing;
  bool intra_broadcast = true;
  bool intra_compress = true;
  bool dummy_compression = false;
  bool remote_buf = true;  // CGX_REMOTE_BUF_COMPRESSION: quantize straight into peer-visible memory. The fused
                           // kernel always does (with proper signalling, unlike the reference's experimental
                           // variant, SURVEY.md §2.8 #7); the variable is accepted for compatibility.
  int lanes = 0;
  int64_t timeout_ms = 120000;
  int local_size = 0;
  uint32_t min_lane_elems = 4096;
  int64_t oneshot_max_bytes = 2 << 20;
  int overlap_lanes = 64;  // lanes of an allreduce issued from the DDP hook (backward still needs the SMs)
  static EngineConfig read();
};

int log_level();
void log_msg(int level, const char* fmt, ...);

}  // namespace cgx
