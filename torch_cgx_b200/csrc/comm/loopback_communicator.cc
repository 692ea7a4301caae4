#include "loopback_communicator.h"

#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <tuple>

#include "symmetric_heap.h"  // cuda_check

namespace cgx {

LoopbackHub::LoopbackHub(int world, int64_t timeout_ms)
    : world_(world), timeout_(timeout_ms), posted_((size_t)world), done_((size_t)world, 0) {}

void LoopbackHub::reset(bool record) {
  std::lock_guard<std::mutex> lk(mu_);
  for (auto& p : posted_) p.clear();
  std::fill(done_.begin(), done_.end(), 0);
  failure_.clear();
  record_ = record;
  messages_.clear();
  barrier_count_ = 0;
}

void LoopbackHub::finish(int rank) {
  std::lock_guard<std::mutex> lk(mu_);
  done_[rank] = 1;
  cv_.notify_all();
}

void LoopbackHub::fail_locked(const std::string& msg) {
  if (failure_.empty()) failure_ = msg.empty() ? "loopback: unknown failure" : msg;
  cv_.notify_all();
}

void LoopbackHub::fail(const std::string& msg) {
  std::lock_guard<std::mutex> lk(mu_);
  fail_locked(msg);
}

bool LoopbackHub::failed() const {
  std::lock_guard<std::mutex> lk(mu_);
  return !failure_.empty();
}

std::string LoopbackHub::failure() const {
  std::lock_guard<std::mutex> lk(mu_);
  return failure_;
}

std::vector<LoopbackHub::Message> LoopbackHub::messages() const {
  std::lock_guard<std::mutex> lk(mu_);
  std::vector<Message> out = messages_;
  std::sort(out.begin(), out.end(), [](const Message& a, const Message& b) {
    return std::tie(a.exchange, a.src, a.dst) < std::tie(b.exchange, b.src, b.dst);
  });
  return out;
}

void LoopbackHub::throw_if_failed() const {
  if (!failure_.empty()) throw std::runtime_error("loopback: released after a failure: " + failure_);
}

template <class Pred>
void LoopbackHub::wait_for(std::unique_lock<std::mutex>& lk, Pred pred, const std::string& what) {
  const bool ok = cv_.wait_for(lk, timeout_, [&] { return !failure_.empty() || pred(); });
  if (!ok) {
    fail_locked("loopback: timed out after " + std::to_string(timeout_.count()) + " ms: " + what);
    throw std::runtime_error(failure_);
  }
  throw_if_failed();
}

const P2POp* LoopbackHub::find(const Posted& p, bool send, int peer, size_t* index) {
  for (size_t i = 0; i < p.ops.size(); ++i)
    if (p.ops[i].send == send && p.ops[i].peer == peer) {
      if (index) *index = i;
      return &p.ops[i];
    }
  return nullptr;
}

void LoopbackHub::exchange(int rank, const std::vector<P2POp>& ops, bool cuda, cudaStream_t stream) {
  // the send data has been produced and the receive buffers are no longer read by earlier work
  if (cuda) cuda_check(cudaStreamSynchronize(stream), "loopback: synchronise before an exchange");
  std::unique_lock<std::mutex> lk(mu_);
  throw_if_failed();
  const size_t e = posted_[rank].size();
  const std::string at = "exchange " + std::to_string(e) + ": ";
  auto die = [&](const std::string& msg) {
    fail_locked("loopback: " + at + msg);
    throw std::runtime_error(failure_);
  };
  for (size_t i = 0; i < ops.size(); ++i) {
    const P2POp& o = ops[i];
    if (o.peer < 0 || o.peer >= world_ || o.peer == rank)
      die("rank " + std::to_string(rank) + " addresses rank " + std::to_string(o.peer));
    for (size_t j = 0; j < i; ++j)
      if (ops[j].send == o.send && ops[j].peer == o.peer)
        die("rank " + std::to_string(rank) + " posts two " + (o.send ? "sends to" : "receives from") + " rank " +
            std::to_string(o.peer));
  }
  posted_[rank].push_back(Posted{ops, std::vector<char>(ops.size(), 0)});
  cv_.notify_all();
  const std::string me = "rank " + std::to_string(rank);
  // a peer that has returned without posting exchange e will never post it
  auto gone = [&](int p) { return done_[p] && posted_[p].size() <= e; };

  // receives: wait until the sender has posted exchange e, then copy its bytes
  for (const P2POp& o : ops) {
    if (o.send) continue;
    const int p = o.peer;
    const std::string who = "rank " + std::to_string(p);
    wait_for(lk, [&] { return posted_[p].size() > e || gone(p); },
             me + " waits for " + who + " to post " + at + "(" + who + " has posted " +
                 std::to_string(posted_[p].size()) + ")");
    if (posted_[p].size() <= e)
      die(me + " expects " + std::to_string(o.bytes) + " bytes from " + who + ", which returned after " +
          std::to_string(posted_[p].size()) + " exchanges");
    size_t si = 0;
    Posted& src = posted_[p][e];
    const P2POp* s = find(src, true, rank, &si);
    if (!s) die(me + " expects " + std::to_string(o.bytes) + " bytes from " + who + ", which sends it nothing");
    if (s->bytes != o.bytes)
      die(who + " sends " + std::to_string(s->bytes) + " bytes to " + me + ", which expects " +
          std::to_string(o.bytes));
    if (o.bytes) {
      if (cuda) {
        // a device-to-device cudaMemcpy returns before the copy has run: copy on the receiver's stream
        // and wait for it, so the bytes have landed (receiver) and been read (sender) once it is consumed
        cuda_check(cudaMemcpyAsync(o.buf, s->buf, o.bytes, cudaMemcpyDeviceToDevice, stream), "loopback: copy");
        cuda_check(cudaStreamSynchronize(stream), "loopback: wait for the copy");
      } else {
        std::memcpy(o.buf, s->buf, o.bytes);
      }
    }
    if (record_) {
      Message m{(int64_t)e, p, rank, std::vector<uint8_t>(o.bytes)};
      if (o.bytes) {
        if (cuda) {
          cuda_check(cudaMemcpyAsync(m.bytes.data(), o.buf, o.bytes, cudaMemcpyDeviceToHost, stream),
                     "loopback: record");
          cuda_check(cudaStreamSynchronize(stream), "loopback: wait for the record");
        } else {
          std::memcpy(m.bytes.data(), o.buf, o.bytes);
        }
      }
      messages_.push_back(std::move(m));
    }
    src.consumed[si] = 1;
    cv_.notify_all();
  }

  // sends: the receiver must post a matching receive of the same size and copy it
  for (size_t i = 0; i < ops.size(); ++i) {
    const P2POp& o = ops[i];
    if (!o.send) continue;
    const int p = o.peer;
    const std::string who = "rank " + std::to_string(p);
    wait_for(lk, [&] { return posted_[p].size() > e || gone(p); },
             me + " waits for " + who + " to post " + at + "(" + who + " has posted " +
                 std::to_string(posted_[p].size()) + ")");
    if (posted_[p].size() <= e)
      die(me + " sends " + std::to_string(o.bytes) + " bytes to " + who + ", which returned after " +
          std::to_string(posted_[p].size()) + " exchanges");
    const P2POp* r = find(posted_[p][e], false, rank, nullptr);
    if (!r) die(me + " sends " + std::to_string(o.bytes) + " bytes to " + who + ", which receives nothing from it");
    if (r->bytes != o.bytes)
      die(me + " sends " + std::to_string(o.bytes) + " bytes to " + who + ", which expects " +
          std::to_string(r->bytes));
    Posted& mine = posted_[rank][e];
    wait_for(lk, [&] { return mine.consumed[i] != 0; }, me + " waits for " + who + " to receive " + at);
  }
}

void LoopbackHub::barrier(int rank) {
  std::unique_lock<std::mutex> lk(mu_);
  throw_if_failed();
  const uint64_t gen = barrier_gen_;
  if (++barrier_count_ == world_) {
    barrier_count_ = 0;
    ++barrier_gen_;
    cv_.notify_all();
    return;
  }
  wait_for(lk, [&] { return barrier_gen_ != gen; }, "rank " + std::to_string(rank) + " waits in a barrier");
}

}  // namespace cgx
