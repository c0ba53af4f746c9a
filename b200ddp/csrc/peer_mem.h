// NVSwitch peer-memory substrate (replacement for ProcessGroupNCCL on the hot path).
//
// Every rank owns one VMM allocation (cuMemCreate, POSIX-FD shareable) - the "arena".  Arenas of all
// ranks are mapped into ONE contiguous VA window per process, rank r at `base + r*stride`, so a
// kernel reaches any peer with pointer arithmetic.  The first kSignalBytes of each arena are signal
// pads for the in-kernel cross-GPU barriers; the rest is staging space handed out by a bump
// allocator (identical offsets on every rank = symmetric memory).  When the device supports
// multicast (NVLS), the arenas are additionally bound to one multicast object and mapped at
// `mc_base`: a store there lands in every GPU's arena, a multimem.ld_reduce sums all copies in
// the switch.
//
// FDs travel between the per-GPU processes over abstract-namespace unix datagram sockets
// (SCM_RIGHTS).  torch.distributed is used by the Python side only as the bootstrap barrier.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

namespace b200 {

constexpr size_t kSignalBytes = 4 << 20;   // 4 MiB of signal pads at the start of every arena
constexpr size_t kPadSetBytes = 32 << 10;  // one PadSet (comm_kernels.cuh) per staging region -> 128 sets
constexpr int kMaxRanks = 8;               // one NVSwitch domain (HGX H100)
constexpr int kMaxCommBlocks = 264;             // 2 light CTAs per SM on 132 SMs

class PeerArena {
 public:
  PeerArena(int rank, int world, int device, size_t bytes, const std::string& uid);
  ~PeerArena();
  PeerArena(const PeerArena&) = delete;

  // bootstrap: bind_socket() on every rank, <host barrier>, exchange(), <host barrier>,
  // setup_multicast_root()/join..., see parallel/peer.py
  void bind_socket();
  void exchange();                 // allocate local arena, swap FDs, map all peers
  bool multicast_supported() const { return mc_supported_; }
  void multicast_create();         // rank 0: create + send FD ; others: receive + import
  void multicast_add_device();     // all ranks
  void multicast_bind();           // all ranks, after everyone added its device
  void disable_multicast();        // agreed fallback
  void close();

  int rank() const { return rank_; }
  int world() const { return world_; }
  int device() const { return device_; }
  size_t bytes() const { return bytes_; }           // usable bytes per rank (incl. signal pads)
  size_t stride() const { return stride_; }
  char* base() const { return base_; }              // VA of rank 0's arena in this process
  char* local() const { return base_ + (size_t)rank_ * stride_; }
  char* peer(int r) const { return base_ + (size_t)r * stride_; }
  char* mc_base() const { return mc_base_; }        // nullptr without multicast
  bool has_multicast() const { return mc_base_ != nullptr; }

  // symmetric bump allocation (same call sequence on every rank -> same offsets)
  size_t alloc(size_t nbytes, size_t align = 256);
  size_t used() const { return bump_; }
  void rewind(size_t mark) { if (mark >= kSignalBytes && mark <= bump_) bump_ = mark; }   // release everything allocated after `mark`

  // device-visible error word (pinned, mapped): kernels write a code on barrier timeout
  volatile int* error_word_host() const { return err_host_; }
  int* error_word_dev() const { return err_dev_; }
  int check_error() const { return err_host_ ? *err_host_ : 0; }
  void clear_error() { if (err_host_) *err_host_ = 0; }

 private:
  void send_fd(int to_rank, int fd, int tag);
  int recv_fd(int* from_rank, int* tag);
  std::string sock_name(int r) const;

  int rank_, world_, device_;
  size_t bytes_ = 0, stride_ = 0, gran_ = 0, bump_ = kSignalBytes;
  std::string uid_;
  int sock_ = -1;
  unsigned long long local_handle_ = 0;
  std::vector<unsigned long long> peer_handles_;
  char* base_ = nullptr;
  char* mc_base_ = nullptr;
  unsigned long long mc_handle_ = 0;
  bool mc_supported_ = false, mc_bound_ = false, mapped_ = false;
  int* err_host_ = nullptr;
  int* err_dev_ = nullptr;
};

}  // namespace b200
