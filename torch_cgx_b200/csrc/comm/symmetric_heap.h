// Symmetric peer-mapped device heap: the H100 replacement for the reference's
// three point-to-point transports. Every rank owns ONE region
//   [sync][flags1][flags2][recv1: W slots][recv2: W slots][one-shot A: W slots][one-shot B: W slots][a2a landed][a2a released]
// and maps every peer's region into its own address space, so kernels move data with ordinary
// ld/st over NVLink 4 / NVSwitch and signal with release/acquire flags -- no host staging, no
// semaphores, no MPI.
//
// Two ways to get there:
//  * VMM (default when the driver allows it): cuMemCreate + POSIX file-descriptor handles passed
//    over unix sockets (comm/fd_channel), and -- when the GPUs sit behind an NVSwitch with
//    multicast enabled -- ONE multicast object bound to every rank's region (cuMulticastCreate /
//    AddDevice / BindMem). The multicast alias lets a kernel write all replicas with a single
//    multimem.st and reduce all replicas inside the switch with multimem.ld_reduce (NVLS).
//  * cudaMalloc + cudaIpc handles: the fallback (CGX_VMM=0, or no driver support).
// Inside one process (tests, single-process multi-stream simulation) plain pointers are shared.
//
// Replaces: SHMCommunicator + shm_utils (POSIX shm + named semaphores + IPC events, GPU->pinned
// host->GPU over PCIe; /root/reference/src/common/shm_communicator.cc:54-330, shm_utils.cc:51-136),
// MPICommunicator (/root/reference/src/common/mpi_communicator.cc:24-84), PersistentBuffer
// (/root/reference/src/common/buffer.cc:23-31) and the NCCL bootstrap
// (/root/reference/src/common/nccl_reduce.cc:52-67). Handles travel through the c10d Store
// (KVStore below) instead of MPI messages.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <string>
#include <vector>

namespace cgx {

struct DeviceSync;

struct HeapLayout {
  int world = 1;
  uint32_t flag_stride = 0;  // lanes capacity (multiple of 32)
  uint32_t slot_bytes = 0;   // bytes per (source rank) slot, multiple of 256
  uint32_t os_slot_bytes = 0;  // per-source slot of the two one-shot regions
  // a2a_landed / a2a_released: the all-to-all's 64-bit window flags, [source * flag_stride + lane]
  size_t sync_off = 0, flags1_off = 0, flags2_off = 0, a2a_landed_off = 0, a2a_released_off = 0, recv1_off = 0, recv2_off = 0, os_off[2] = {0, 0}, total = 0;
  // throws std::invalid_argument when a slot size does not fit the 32-bit offsets kernels use
  static HeapLayout make(int world, int max_lanes, size_t slot_bytes, size_t os_slot_bytes = 0);
};

// Minimal key-value rendezvous (implemented over c10d::Store by the backend,
// over a std::map by in-process tests).
class KVStore {
 public:
  virtual ~KVStore() = default;
  virtual void set(const std::string& key, const std::vector<uint8_t>& value) = 0;
  virtual std::vector<uint8_t> get(const std::string& key) = 0;  // blocks until present
};

enum class HeapKind { kNone, kCudaMalloc, kVmm };

class SymmetricHeap {
 public:
  SymmetricHeap(int rank, int world, const HeapLayout& layout);
  ~SymmetricHeap();
  SymmetricHeap(const SymmetricHeap&) = delete;
  SymmetricHeap& operator=(const SymmetricHeap&) = delete;

  // peers live in this process (tests / single-process multi-stream simulation)
  void connect_local(const std::vector<SymmetricHeap*>& all);
  // one process per GPU: agree on VMM(+multicast) or cudaIpc, allocate, exchange handles
  void connect_ipc(KVStore& store, const std::string& prefix);

  int rank() const { return rank_; }
  int world() const { return world_; }
  int device() const { return device_; }
  const HeapLayout& layout() const { return layout_; }
  bool connected() const { return connected_; }
  HeapKind kind() const { return kind_; }
  bool has_multicast() const { return mc_base_ != nullptr; }

  uint8_t* base(int peer) const { return bases_[peer]; }
  uint8_t* recv1(int peer) const { return bases_[peer] + layout_.recv1_off; }
  uint8_t* recv2(int peer) const { return bases_[peer] + layout_.recv2_off; }
  uint8_t* oneshot(int peer, int parity) const { return bases_[peer] + layout_.os_off[parity & 1]; }
  uint32_t* flags1(int peer) const { return reinterpret_cast<uint32_t*>(bases_[peer] + layout_.flags1_off); }
  uint32_t* flags2(int peer) const { return reinterpret_cast<uint32_t*>(bases_[peer] + layout_.flags2_off); }
  uint64_t* a2a_landed(int peer) const { return reinterpret_cast<uint64_t*>(bases_[peer] + layout_.a2a_landed_off); }
  uint64_t* a2a_released(int peer) const {
    return reinterpret_cast<uint64_t*>(bases_[peer] + layout_.a2a_released_off);
  }
  // multicast aliases (nullptr without NVLS)
  uint8_t* mc_recv1() const { return mc_base_ ? mc_base_ + layout_.recv1_off : nullptr; }
  uint8_t* mc_recv2() const { return mc_base_ ? mc_base_ + layout_.recv2_off : nullptr; }
  uint8_t* mc_oneshot(int parity) const { return mc_base_ ? mc_base_ + layout_.os_off[parity & 1] : nullptr; }
  DeviceSync* sync_device() const { return reinterpret_cast<DeviceSync*>(bases_[rank_] + layout_.sync_off); }

  // host-visible error word written by kernels on timeout (word 0) and the abort request the
  // host raises to make every spinning kernel of this heap give up (word 1)
  uint32_t* status_device() const { return status_dev_; }
  const uint32_t* abort_device() const { return status_dev_ + 1; }
  uint32_t status_host() const { return status_host_ ? *(volatile uint32_t*)status_host_ : 0; }
  void clear_status() { if (status_host_) *(volatile uint32_t*)status_host_ = 0; }
  void request_abort(bool on) { if (status_host_) *((volatile uint32_t*)status_host_ + 1) = on ? 1u : 0u; }

 private:
  void alloc_cuda_malloc();
  void connect_cuda_ipc(KVStore& store, const std::string& prefix, const std::vector<bool>& same_process,
                        const std::vector<uint64_t>& local_ptrs);
  bool connect_vmm(KVStore& store, const std::string& prefix, bool want_multicast);
  void release_vmm();

  int rank_, world_, device_ = 0;
  HeapLayout layout_;
  HeapKind kind_ = HeapKind::kNone;
  std::vector<uint8_t*> bases_;   // [world]; bases_[rank_] is the local allocation
  std::vector<bool> ipc_opened_;
  uint8_t* mc_base_ = nullptr;
  // VMM bookkeeping (driver handles kept as integers to keep cuda.h out of this header)
  size_t vmm_size_ = 0;
  std::vector<unsigned long long> vmm_handles_;  // [world] imported / own allocation handles
  unsigned long long mc_handle_ = 0;
  bool mc_bound_ = false;
  uint32_t* status_host_ = nullptr;
  uint32_t* status_dev_ = nullptr;
  bool connected_ = false;
};

void cuda_check(cudaError_t e, const char* what);

// 128-bit random token generated once per process: identifies "same process" reliably
// (PIDs repeat across hosts, containers and PID namespaces).
const uint8_t* process_token();

}  // namespace cgx
