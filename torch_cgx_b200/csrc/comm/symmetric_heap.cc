#include "symmetric_heap.h"

#include <cuda.h>
#include <unistd.h>

#include <chrono>
#include <cstring>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>

#include "../common/config.h"
#include "../kernels/launch.h"
#include "fd_channel.h"

namespace cgx {

void cuda_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    std::string msg = std::string("cgx: CUDA error in ") + what + ": " + cudaGetErrorString(e);
    throw std::runtime_error(msg);
  }
}

const uint8_t* process_token() {
  static uint8_t token[16];
  static bool init = [] {
    std::random_device rd;
    for (int i = 0; i < 16; i += 4) {
      const uint32_t v = rd();
      std::memcpy(token + i, &v, 4);
    }
    // mix in pid + time so that a deterministic random_device still separates processes
    const uint64_t salt = ((uint64_t)getpid() << 32) ^
                          (uint64_t)std::chrono::high_resolution_clock::now().time_since_epoch().count();
    for (int i = 0; i < 8; ++i) token[i] ^= (uint8_t)(salt >> (8 * i));
    return true;
  }();
  (void)init;
  return token;
}

static size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

HeapLayout HeapLayout::make(int world, int max_lanes, size_t slot_bytes, size_t os_slot_bytes) {
  HeapLayout l;
  l.world = world;
  l.flag_stride = (uint32_t)round_up((size_t)(max_lanes < 1 ? 1 : max_lanes), 32);
  const size_t slot = round_up(slot_bytes < 256 ? 256 : slot_bytes, 256);
  const size_t os_slot = round_up(os_slot_bytes, 256);
  // kernels address with 32-bit offsets inside a region: W slots (x2 for the one-shot pair)
  if (slot * (size_t)world >= (1ull << 32) || 2 * os_slot * (size_t)world >= (1ull << 32))
    throw std::invalid_argument(
        "cgx: symmetric heap slots exceed 4 GiB per region (lower CGX_FUSION_BUFFER_SIZE_MB / CGX_ONESHOT_MAX_BYTES)");
  l.slot_bytes = (uint32_t)slot;
  l.os_slot_bytes = (uint32_t)os_slot;
  const size_t flags_bytes = round_up((size_t)world * l.flag_stride * sizeof(uint32_t), 256);
  l.sync_off = 0;
  l.flags1_off = 256;
  l.flags2_off = l.flags1_off + flags_bytes;
  l.recv1_off = l.flags2_off + flags_bytes;
  l.recv2_off = l.recv1_off + (size_t)world * slot;
  l.os_off[0] = l.recv2_off + (size_t)world * slot;
  l.os_off[1] = l.os_off[0] + (size_t)world * os_slot;
  // the all-to-all's flags go last, so every region the other kernels use keeps its offset
  const size_t flags64_bytes = round_up((size_t)world * l.flag_stride * sizeof(uint64_t), 256);
  l.a2a_landed_off = l.os_off[1] + (size_t)world * os_slot;
  l.a2a_released_off = l.a2a_landed_off + flags64_bytes;
  l.total = l.a2a_released_off + flags64_bytes;
  return l;
}

// ---------------------------------------------------------------------------------------------
// CUDA driver entry points, resolved at run time (the extension must load on machines without
// a driver: the CPU test tier imports it)
// ---------------------------------------------------------------------------------------------
namespace {

struct DriverApi {
  bool ok = false;
  CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType,
                                         unsigned long long) = nullptr;
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t,
                               unsigned long long) = nullptr;
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
  CUresult (*MulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t) = nullptr;
};

template <typename F>
bool load_sym(const char* name, F* out) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult st;
  if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &st) != cudaSuccess || st != cudaDriverEntryPointSuccess ||
      fn == nullptr) {
    (void)cudaGetLastError();
    return false;
  }
  *out = reinterpret_cast<F>(fn);
  return true;
}

const DriverApi& driver() {
  static DriverApi api = [] {
    DriverApi a;
    bool ok = true;
    ok &= load_sym("cuGetErrorString", &a.GetErrorString);
    ok &= load_sym("cuDeviceGet", &a.DeviceGet);
    ok &= load_sym("cuDeviceGetAttribute", &a.DeviceGetAttribute);
    ok &= load_sym("cuMemCreate", &a.MemCreate);
    ok &= load_sym("cuMemRelease", &a.MemRelease);
    ok &= load_sym("cuMemAddressReserve", &a.MemAddressReserve);
    ok &= load_sym("cuMemAddressFree", &a.MemAddressFree);
    ok &= load_sym("cuMemMap", &a.MemMap);
    ok &= load_sym("cuMemUnmap", &a.MemUnmap);
    ok &= load_sym("cuMemSetAccess", &a.MemSetAccess);
    ok &= load_sym("cuMemGetAllocationGranularity", &a.MemGetAllocationGranularity);
    ok &= load_sym("cuMemExportToShareableHandle", &a.MemExportToShareableHandle);
    ok &= load_sym("cuMemImportFromShareableHandle", &a.MemImportFromShareableHandle);
    // multicast is optional (driver >= 12.1)
    bool mc = true;
    mc &= load_sym("cuMulticastCreate", &a.MulticastCreate);
    mc &= load_sym("cuMulticastAddDevice", &a.MulticastAddDevice);
    mc &= load_sym("cuMulticastBindMem", &a.MulticastBindMem);
    mc &= load_sym("cuMulticastGetGranularity", &a.MulticastGetGranularity);
    mc &= load_sym("cuMulticastUnbind", &a.MulticastUnbind);
    if (!mc) a.MulticastCreate = nullptr;
    a.ok = ok;
    return a;
  }();
  return api;
}

std::string cu_err(CUresult r) {
  const char* s = nullptr;
  if (driver().GetErrorString && driver().GetErrorString(r, &s) == CUDA_SUCCESS && s) return s;
  return "CUresult " + std::to_string((int)r);
}

#define CU_TRY(expr, what)                                                        \
  do {                                                                            \
    CUresult r_ = (expr);                                                         \
    if (r_ != CUDA_SUCCESS) {                                                     \
      log_msg(1, "cgx: %s failed: %s", what, cu_err(r_).c_str());                 \
      return false;                                                               \
    }                                                                             \
  } while (0)

struct HeapHello {
  uint8_t token[16];
  char host[64];
  uint64_t total;
  int32_t device;
  int32_t vmm_ok;
  int32_t mc_ok;
  int32_t pad;
};

struct IpcHello {
  cudaIpcMemHandle_t handle;
  uint64_t local_ptr;  // valid only inside the same process
};

template <typename S>
std::vector<uint8_t> to_blob(const S& s) {
  std::vector<uint8_t> b(sizeof(S));
  std::memcpy(b.data(), &s, sizeof(S));
  return b;
}
template <typename S>
S from_blob(const std::vector<uint8_t>& b, const char* what) {
  if (b.size() != sizeof(S)) throw std::runtime_error(std::string("cgx: malformed ") + what + " from peer");
  S s;
  std::memcpy(&s, b.data(), sizeof(S));
  return s;
}

// collective AND over the group: every rank learns whether every rank succeeded at `step`
bool agree(KVStore& store, const std::string& prefix, const std::string& step, int rank, int world, bool ok) {
  store.set(prefix + "/" + step + "/" + std::to_string(rank), {(uint8_t)(ok ? 1 : 0)});
  bool all = ok;
  for (int p = 0; p < world; ++p) {
    if (p == rank) continue;
    const std::vector<uint8_t> v = store.get(prefix + "/" + step + "/" + std::to_string(p));
    all = all && !v.empty() && v[0] == 1;
  }
  return all;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
SymmetricHeap::SymmetricHeap(int rank, int world, const HeapLayout& layout)
    : rank_(rank), world_(world), layout_(layout), bases_(world, nullptr), ipc_opened_(world, false),
      vmm_handles_(world, 0ull) {
  cuda_check(cudaGetDevice(&device_), "cudaGetDevice");
  void* h = nullptr;
  cuda_check(cudaHostAlloc(&h, 64, cudaHostAllocMapped), "cudaHostAlloc(status)");
  std::memset(h, 0, 64);
  status_host_ = static_cast<uint32_t*>(h);
  void* d = nullptr;
  cuda_check(cudaHostGetDevicePointer(&d, h, 0), "cudaHostGetDevicePointer(status)");
  status_dev_ = static_cast<uint32_t*>(d);
  if (world_ == 1) {
    alloc_cuda_malloc();
    connected_ = true;
  }
}

void SymmetricHeap::alloc_cuda_malloc() {
  void* p = nullptr;
  cuda_check(cudaMalloc(&p, layout_.total), "cudaMalloc(symmetric heap)");
  cuda_check(cudaMemset(p, 0, layout_.total), "cudaMemset(symmetric heap)");
  cuda_check(cudaDeviceSynchronize(), "heap init sync");
  bases_[rank_] = static_cast<uint8_t*>(p);
  kind_ = HeapKind::kCudaMalloc;
}

void SymmetricHeap::release_vmm() {
  const DriverApi& d = driver();
  if (!d.ok) return;
  if (mc_base_) {
    d.MemUnmap((CUdeviceptr)mc_base_, vmm_size_);
    d.MemAddressFree((CUdeviceptr)mc_base_, vmm_size_);
    mc_base_ = nullptr;
  }
  if (mc_handle_) {
    if (mc_bound_ && d.MulticastUnbind) {
      CUdevice dev;
      if (d.DeviceGet(&dev, device_) == CUDA_SUCCESS) d.MulticastUnbind(mc_handle_, dev, 0, vmm_size_);
    }
    d.MemRelease(mc_handle_);
    mc_handle_ = 0;
    mc_bound_ = false;
  }
  for (int p = 0; p < world_; ++p) {
    if (bases_[p] && vmm_handles_[p]) {
      d.MemUnmap((CUdeviceptr)bases_[p], vmm_size_);
      d.MemAddressFree((CUdeviceptr)bases_[p], vmm_size_);
      bases_[p] = nullptr;
    }
    if (vmm_handles_[p]) {
      d.MemRelease(vmm_handles_[p]);
      vmm_handles_[p] = 0;
    }
  }
  kind_ = HeapKind::kNone;
}

SymmetricHeap::~SymmetricHeap() {
  if (kind_ == HeapKind::kVmm) {
    release_vmm();
  } else {
    for (int p = 0; p < world_; ++p)
      if (p != rank_ && ipc_opened_[p] && bases_[p]) cudaIpcCloseMemHandle(bases_[p]);
    if (bases_[rank_]) cudaFree(bases_[rank_]);
  }
  if (status_host_) cudaFreeHost(status_host_);
}

void SymmetricHeap::connect_local(const std::vector<SymmetricHeap*>& all) {
  if ((int)all.size() != world_) throw std::invalid_argument("cgx: connect_local needs one heap per rank");
  if (bases_[rank_] == nullptr) alloc_cuda_malloc();
  for (int p = 0; p < world_; ++p) {
    if (p == rank_) continue;
    if (all[p]->layout_.total != layout_.total) throw std::invalid_argument("cgx: heap layouts differ");
    if (all[p]->bases_[p] == nullptr) all[p]->alloc_cuda_malloc();
    bases_[p] = all[p]->bases_[p];
    if (all[p]->device_ != device_) {
      int can = 0;
      cuda_check(cudaDeviceCanAccessPeer(&can, device_, all[p]->device_), "cudaDeviceCanAccessPeer");
      if (!can) throw std::runtime_error("cgx: no P2P access between in-process devices");
      cudaError_t e = cudaDeviceEnablePeerAccess(all[p]->device_, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) cuda_check(e, "cudaDeviceEnablePeerAccess");
      (void)cudaGetLastError();
    }
  }
  connected_ = true;
}

void SymmetricHeap::connect_ipc(KVStore& store, const std::string& prefix) {
  // ---- who is out there, and what can everybody do?
  HeapHello me;
  std::memset(&me, 0, sizeof(me));
  std::memcpy(me.token, process_token(), 16);
  if (gethostname(me.host, sizeof(me.host) - 1) != 0) me.host[0] = 0;
  me.total = layout_.total;
  me.device = device_;
  {
    const DriverApi& d = driver();
    int vmm = 0, mc = 0;
    CUdevice dev;
    if (d.ok && env_bool("CGX_VMM", true) && d.DeviceGet(&dev, device_) == CUDA_SUCCESS) {
      d.DeviceGetAttribute(&vmm, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev);
      if (vmm && d.MulticastCreate && env_bool("CGX_NVLS", true))
        d.DeviceGetAttribute(&mc, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev);
    }
    me.vmm_ok = vmm;
    me.mc_ok = mc;
  }
  store.set(prefix + "/hello/" + std::to_string(rank_), to_blob(me));
  std::vector<bool> same_process(world_, false);
  bool all_vmm = me.vmm_ok != 0, all_mc = me.mc_ok != 0, any_same = false;
  for (int p = 0; p < world_; ++p) {
    if (p == rank_) continue;
    const HeapHello other = from_blob<HeapHello>(store.get(prefix + "/hello/" + std::to_string(p)), "heap hello");
    if (other.total != layout_.total)
      throw std::runtime_error(
          "cgx: peer heap layout differs (CGX_FUSION_BUFFER_SIZE_MB / CGX_LANES must match on all ranks)");
    if (std::strncmp(other.host, me.host, sizeof(me.host)) != 0)
      throw std::runtime_error(std::string("cgx: rank ") + std::to_string(p) + " of this node group runs on host '" +
                               other.host + "' but this rank runs on '" + me.host +
                               "': peer memory only works inside one node -- set LOCAL_WORLD_SIZE / CGX_LOCAL_SIZE "
                               "to the number of ranks per node");
    same_process[p] = std::memcmp(other.token, me.token, 16) == 0;
    any_same = any_same || same_process[p];
    all_vmm = all_vmm && other.vmm_ok != 0;
    all_mc = all_mc && other.mc_ok != 0;
  }

  bool done = false;
  if (all_vmm && !any_same) {
    done = connect_vmm(store, prefix, all_mc);
    if (!done) log_msg(1, "cgx[%d]: VMM heap setup failed on some rank, falling back to cudaMalloc + cudaIpc", rank_);
  }
  if (!done) {
    alloc_cuda_malloc();
    IpcHello ih;
    std::memset(&ih, 0, sizeof(ih));
    cuda_check(cudaIpcGetMemHandle(&ih.handle, bases_[rank_]), "cudaIpcGetMemHandle");
    ih.local_ptr = (uint64_t)(uintptr_t)bases_[rank_];
    store.set(prefix + "/ipc/" + std::to_string(rank_), to_blob(ih));
    for (int p = 0; p < world_; ++p) {
      if (p == rank_) continue;
      const IpcHello other = from_blob<IpcHello>(store.get(prefix + "/ipc/" + std::to_string(p)), "ipc handle");
      if (same_process[p]) {
        bases_[p] = reinterpret_cast<uint8_t*>((uintptr_t)other.local_ptr);
        continue;
      }
      void* ptr = nullptr;
      cudaError_t e = cudaIpcOpenMemHandle(&ptr, other.handle, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        std::string msg = "cgx: cudaIpcOpenMemHandle(rank " + std::to_string(p) + ") failed: " +
                          cudaGetErrorString(e) +
                          " -- the fused P2P path needs NVLink/PCIe peer access between all local GPUs";
        (void)cudaGetLastError();
        throw std::runtime_error(msg);
      }
      bases_[p] = static_cast<uint8_t*>(ptr);
      ipc_opened_[p] = true;
    }
  }
  // everybody has mapped everybody before anyone starts writing flags
  (void)agree(store, prefix, "ready", rank_, world_, true);
  connected_ = true;
  log_msg(1, "cgx[%d]: symmetric heap connected (%s%s, %.1f MB per rank)", rank_,
          kind_ == HeapKind::kVmm ? "VMM + fd handles" : "cudaMalloc + cudaIpc", mc_base_ ? " + NVLS multicast" : "",
          (double)layout_.total / (1 << 20));
}

// VMM allocation, descriptor exchange, peer mappings and (optionally) the multicast object.
// Every step that can fail is followed by a collective agreement, so either every rank ends up
// with the same kind of heap or every rank falls back together.
bool SymmetricHeap::connect_vmm(KVStore& store, const std::string& prefix, bool want_multicast) {
  const DriverApi& d = driver();
  CUdevice dev;
  CUmemAllocationProp prop;
  std::memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device_;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  CUmemAccessDesc access;
  std::memset(&access, 0, sizeof(access));
  access.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  access.location.id = device_;
  access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  CUmulticastObjectProp mcprop;
  std::memset(&mcprop, 0, sizeof(mcprop));
  mcprop.numDevices = (unsigned)world_;
  mcprop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;

  std::unique_ptr<FdChannel> chan;
  int my_fd = -1;
  size_t gran = 0;

  // ---- stage A: my allocation, mapped and zeroed
  auto stage_a = [&]() -> bool {
    CU_TRY(d.DeviceGet(&dev, device_), "cuDeviceGet");
    CU_TRY(d.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED),
           "cuMemGetAllocationGranularity");
    size_t size = round_up(layout_.total, gran);
    if (want_multicast) {
      size_t mg = 0;
      mcprop.size = size;
      if (d.MulticastGetGranularity(&mg, &mcprop, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && mg > 0)
        size = round_up(size, mg);
      else
        want_multicast = false;
    }
    vmm_size_ = size;
    CUmemGenericAllocationHandle h = 0;
    CU_TRY(d.MemCreate(&h, size, &prop, 0), "cuMemCreate");
    vmm_handles_[rank_] = h;
    CUdeviceptr va = 0;
    CU_TRY(d.MemAddressReserve(&va, size, gran, 0, 0), "cuMemAddressReserve");
    bases_[rank_] = reinterpret_cast<uint8_t*>(va);
    CU_TRY(d.MemMap(va, size, 0, h, 0), "cuMemMap");
    CU_TRY(d.MemSetAccess(va, size, &access, 1), "cuMemSetAccess");
    if (cudaMemset(bases_[rank_], 0, size) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
      (void)cudaGetLastError();
      return false;
    }
    CU_TRY(d.MemExportToShareableHandle(&my_fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0),
           "cuMemExportToShareableHandle");
    try {
      chan = std::make_unique<FdChannel>("heap" + std::to_string(rank_));
    } catch (const std::exception& e) {
      log_msg(1, "%s", e.what());
      return false;
    }
    return true;
  };
  kind_ = HeapKind::kVmm;  // release_vmm() cleans up whatever stage A/B left behind
  bool ok = stage_a();
  // the multicast decision must be unanimous as well (granularity query may have failed somewhere)
  const bool mc_wanted = agree(store, prefix, "vmmA_mc", rank_, world_, ok && want_multicast);
  if (!agree(store, prefix, "vmmA", rank_, world_, ok)) {
    if (my_fd >= 0) ::close(my_fd);
    release_vmm();
    return false;
  }

  // ---- stage B: descriptors travel over unix sockets, names over the store
  enum : int32_t { kMsgMem = 1, kMsgMc = 2 };
  {
    const std::string nm = chan->name();
    store.set(prefix + "/chan/" + std::to_string(rank_), std::vector<uint8_t>(nm.begin(), nm.end()));
  }
  std::vector<std::string> names(world_);
  for (int p = 0; p < world_; ++p) {
    if (p == rank_) continue;
    const std::vector<uint8_t> v = store.get(prefix + "/chan/" + std::to_string(p));
    names[p] = std::string(v.begin(), v.end());
  }
  std::vector<FdMessage> inbox;
  // sends never block; while a peer's queue is full we drain our own
  auto exchange = [&](std::vector<std::pair<int, int>> sends /* (peer, fd) */, int32_t kind, size_t expect) -> bool {
    const auto t0 = std::chrono::steady_clock::now();
    size_t got = 0;
    for (const FdMessage& m : inbox) got += m.kind == kind;
    try {
      while (!sends.empty() || got < expect) {
        bool progress = false;
        for (size_t i = 0; i < sends.size();) {
          if (chan->try_send(names[sends[i].first], sends[i].second, kind, rank_)) {
            sends.erase(sends.begin() + i);
            progress = true;
          } else {
            ++i;
          }
        }
        FdMessage m;
        while (chan->try_recv(&m, progress ? 0 : 20)) {
          inbox.push_back(m);
          got += m.kind == kind;
          progress = true;
          if (got >= expect && sends.empty()) break;
        }
        if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(120)) {
          log_msg(1, "cgx[%d]: timed out exchanging memory descriptors", rank_);
          return false;
        }
      }
    } catch (const std::exception& e) {
      log_msg(1, "%s", e.what());
      return false;
    }
    return true;
  };
  auto stage_b = [&]() -> bool {
    std::vector<std::pair<int, int>> sends;
    for (int p = 0; p < world_; ++p)
      if (p != rank_) sends.emplace_back(p, my_fd);
    if (!exchange(sends, kMsgMem, (size_t)world_ - 1)) return false;
    for (FdMessage& m : inbox) {
      if (m.kind != kMsgMem || m.fd < 0) continue;
      const int p = m.src;
      if (p < 0 || p >= world_ || p == rank_ || vmm_handles_[p]) continue;
      CUmemGenericAllocationHandle h = 0;
      CU_TRY(d.MemImportFromShareableHandle(&h, (void*)(uintptr_t)m.fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR),
             "cuMemImportFromShareableHandle");
      vmm_handles_[p] = h;
      ::close(m.fd);
      m.fd = -1;
      CUdeviceptr va = 0;
      CU_TRY(d.MemAddressReserve(&va, vmm_size_, gran, 0, 0), "cuMemAddressReserve(peer)");
      bases_[p] = reinterpret_cast<uint8_t*>(va);
      CU_TRY(d.MemMap(va, vmm_size_, 0, h, 0), "cuMemMap(peer)");
      CU_TRY(d.MemSetAccess(va, vmm_size_, &access, 1), "cuMemSetAccess(peer)");
    }
    for (int p = 0; p < world_; ++p)
      if (bases_[p] == nullptr) return false;
    return true;
  };
  ok = stage_b();
  if (my_fd >= 0) ::close(my_fd);
  my_fd = -1;
  if (!agree(store, prefix, "vmmB", rank_, world_, ok)) {
    for (FdMessage& m : inbox)
      if (m.fd >= 0) ::close(m.fd);
    release_vmm();
    return false;
  }

  // ---- stage C (optional): one multicast object over everybody's allocation
  if (mc_wanted) {
    int mc_fd = -1;
    auto mc_cleanup = [&]() {
      if (mc_base_) {
        d.MemUnmap((CUdeviceptr)mc_base_, vmm_size_);
        d.MemAddressFree((CUdeviceptr)mc_base_, vmm_size_);
        mc_base_ = nullptr;
      }
      if (mc_handle_) {
        if (mc_bound_) d.MulticastUnbind(mc_handle_, dev, 0, vmm_size_);
        d.MemRelease(mc_handle_);
        mc_handle_ = 0;
        mc_bound_ = false;
      }
    };
    auto c0 = [&]() -> bool {  // rank 0 creates and exports, everyone imports
      mcprop.size = vmm_size_;
      if (rank_ == 0) {
        CUmemGenericAllocationHandle mh = 0;
        CU_TRY(d.MulticastCreate(&mh, &mcprop), "cuMulticastCreate");
        mc_handle_ = mh;
        CU_TRY(d.MemExportToShareableHandle(&mc_fd, mh, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0),
               "cuMemExportToShareableHandle(multicast)");
      }
      return true;
    };
    bool mc_ok = agree(store, prefix, "mc0", rank_, world_, c0());
    if (mc_ok) {
      auto c1 = [&]() -> bool {
        std::vector<std::pair<int, int>> sends;
        if (rank_ == 0)
          for (int p = 1; p < world_; ++p) sends.emplace_back(p, mc_fd);
        if (!exchange(sends, kMsgMc, rank_ == 0 ? 0 : 1)) return false;
        if (rank_ != 0) {
          for (FdMessage& m : inbox) {
            if (m.kind != kMsgMc || m.fd < 0) continue;
            CUmemGenericAllocationHandle mh = 0;
            CU_TRY(d.MemImportFromShareableHandle(&mh, (void*)(uintptr_t)m.fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR),
                   "cuMemImportFromShareableHandle(multicast)");
            mc_handle_ = mh;
            ::close(m.fd);
            m.fd = -1;
          }
          if (!mc_handle_) return false;
        }
        CU_TRY(d.MulticastAddDevice(mc_handle_, dev), "cuMulticastAddDevice");
        return true;
      };
      mc_ok = agree(store, prefix, "mc1", rank_, world_, c1());
    }
    if (mc_fd >= 0) ::close(mc_fd);
    if (mc_ok) {
      // every device has been added: binding is allowed now
      auto c2 = [&]() -> bool {
        CU_TRY(d.MulticastBindMem(mc_handle_, 0, vmm_handles_[rank_], 0, vmm_size_, 0), "cuMulticastBindMem");
        mc_bound_ = true;
        CUdeviceptr va = 0;
        CU_TRY(d.MemAddressReserve(&va, vmm_size_, gran, 0, 0), "cuMemAddressReserve(multicast)");
        mc_base_ = reinterpret_cast<uint8_t*>(va);
        CU_TRY(d.MemMap(va, vmm_size_, 0, mc_handle_, 0), "cuMemMap(multicast)");
        CU_TRY(d.MemSetAccess(va, vmm_size_, &access, 1), "cuMemSetAccess(multicast)");
        return true;
      };
      mc_ok = agree(store, prefix, "mc2", rank_, world_, c2());
    }
    if (!mc_ok) {
      log_msg(1, "cgx[%d]: NVLS multicast unavailable, using unicast peer stores", rank_);
      mc_cleanup();
    }
  }
  for (FdMessage& m : inbox)
    if (m.fd >= 0) ::close(m.fd);
  return true;
}

}  // namespace cgx
