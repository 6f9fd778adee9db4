// pybind11 surface of the data-plane extension `torchft_b200._K`.
//
// Design: Python owns policy (which buffers, which peers, which stream); this
// module owns mechanism (peer-memory handles, status block, kernel launches).
// All pointers/streams cross the boundary as integers, so there is no torch
// ABI dependency and the module imports on a CPU-only box (calls then raise).
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "api.h"
#include "audit.cuh"
#include "common.cuh"
#include "zero1.cuh"

namespace py = pybind11;
using namespace tft;

namespace {

inline cudaStream_t S(uintptr_t s) { return reinterpret_cast<cudaStream_t>(s); }
template <typename T = void>
inline T* P(uintptr_t p) { return reinterpret_cast<T*>(p); }

// Host-pinned, device-mapped status block (abort flag, error latch, timeout).
class Status {
 public:
  Status() {
    TFT_CUDA_CHECK(cudaHostAlloc(&host_, sizeof(StatusBlock), cudaHostAllocMapped | cudaHostAllocPortable));
    std::memset((void*)host_, 0, sizeof(StatusBlock));
    host_->timeout_ns = 60ull * 1000 * 1000 * 1000;
    void* d = nullptr;
    TFT_CUDA_CHECK(cudaHostGetDevicePointer(&d, (void*)host_, 0));
    dev_ = reinterpret_cast<StatusBlock*>(d);
  }
  ~Status() {
    if (host_) cudaFreeHost((void*)host_);
  }
  uintptr_t dev_ptr() const { return reinterpret_cast<uintptr_t>(dev_); }
  void set_abort(bool v) { host_->abort = v ? 1u : 0u; }
  bool aborted() const { return host_->abort != 0; }
  py::tuple error() const { return py::make_tuple(host_->error, host_->error_rank, host_->error_seq); }
  void clear() {
    host_->abort = 0;
    host_->error = 0;
    host_->error_rank = 0;
    host_->error_seq = 0;
  }
  // Verdict of commit `seq` written by zero1_commit_kernel: -1 = not there (yet), else 0 / 1.
  int verdict(uint32_t seq) const {
    const uint32_t v = host_->verdict[seq & (kVerdictRing - 1)];
    return (v >> 1) == (seq & 0x7fffffffu) ? (int)(v & 1u) : -1;
  }
  // Global gradient norm the clipping commit kernel posted for `seq` (valid once verdict(seq) is not -1).
  float grad_norm(uint32_t seq) const { return host_->gnorm[seq & (kVerdictRing - 1)]; }
  // Why the token-mean commit kernel vetoed `seq` (zero1::kVetoRows bits; valid once verdict(seq) is not -1).
  uint32_t reason(uint32_t seq) const { return host_->reason[seq & (kVerdictRing - 1)]; }
  void set_timeout_ms(double ms) { host_->timeout_ns = (uint64_t)(ms * 1e6); }
  double timeout_ms() const { return (double)host_->timeout_ns / 1e6; }
  StatusBlock* dev() const { return dev_; }

 private:
  StatusBlock* host_ = nullptr;
  StatusBlock* dev_ = nullptr;
};

// Host-pinned, device-mapped words a kernel writes and the host reads without a copy (the audit report).
class MappedWords {
 public:
  explicit MappedWords(size_t n) : n_(n) {
    TFT_CUDA_CHECK(cudaHostAlloc(&host_, n * 8, cudaHostAllocMapped | cudaHostAllocPortable));
    std::memset((void*)host_, 0, n * 8);
    void* d = nullptr;
    TFT_CUDA_CHECK(cudaHostGetDevicePointer(&d, (void*)host_, 0));
    dev_ = reinterpret_cast<unsigned long long*>(d);
  }
  ~MappedWords() {
    if (host_) cudaFreeHost((void*)host_);
  }
  MappedWords(const MappedWords&) = delete;
  MappedWords& operator=(const MappedWords&) = delete;
  uintptr_t dev_ptr() const { return reinterpret_cast<uintptr_t>(dev_); }
  size_t size() const { return n_; }
  // the words as little-endian bytes (a snapshot; the caller orders it after the kernel that wrote them)
  py::bytes read() const { return py::bytes(reinterpret_cast<const char*>(const_cast<unsigned long long*>(host_)), n_ * 8); }

 private:
  size_t n_;
  volatile unsigned long long* host_ = nullptr;
  unsigned long long* dev_ = nullptr;
};

class PeerTableH {
 public:
  PeerTableH(const std::vector<uintptr_t>& data, const std::vector<uintptr_t>& pads, int rank, int world) {
    if (world < 1 || world > kMaxRanks) throw std::runtime_error("PeerTable: world must be in [1, 8]");
    if ((int)data.size() != world || (int)pads.size() != world)
      throw std::runtime_error("PeerTable: need one data and one pad pointer per rank");
    if (rank < 0 || rank >= world) throw std::runtime_error("PeerTable: bad rank");
    std::memset(&pt, 0, sizeof(pt));
    for (int i = 0; i < world; ++i) {
      pt.data[i] = P<void>(data[i]);
      pt.pads[i] = P<SignalPad>(pads[i]);
    }
    pt.rank = rank;
    pt.world = world;
    pt.timeout_ns = 60ull * 1000 * 1000 * 1000;
  }
  void set_timeout_ms(double ms) { pt.timeout_ns = (uint64_t)(ms * 1e6); }
  // Same peers/pads, different data segment (e.g. a registered gradient buffer).
  PeerTableH with_data(const std::vector<uintptr_t>& data) const {
    PeerTableH o(*this);
    if ((int)data.size() != pt.world) throw std::runtime_error("with_data: wrong number of pointers");
    for (int i = 0; i < pt.world; ++i) o.pt.data[i] = P<void>(data[i]);
    return o;
  }
  int rank() const { return pt.rank; }
  int world() const { return pt.world; }
  PeerTable pt;
};

py::bytes ipc_get_handle(uintptr_t ptr) {
  cudaIpcMemHandle_t h;
  TFT_CUDA_CHECK(cudaIpcGetMemHandle(&h, P<void>(ptr)));
  return py::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
}

uintptr_t ipc_open_handle(const std::string& b) {
  if (b.size() != sizeof(cudaIpcMemHandle_t)) throw std::runtime_error("bad IPC handle size");
  cudaIpcMemHandle_t h;
  std::memcpy(&h, b.data(), sizeof(h));
  void* p = nullptr;
  TFT_CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  return reinterpret_cast<uintptr_t>(p);
}

void ipc_close_handle(uintptr_t p) { TFT_CUDA_CHECK(cudaIpcCloseMemHandle(P<void>(p))); }

uintptr_t symm_alloc(size_t nbytes) {
  void* p = nullptr;
  TFT_CUDA_CHECK(cudaMalloc(&p, nbytes));
  TFT_CUDA_CHECK(cudaMemset(p, 0, nbytes));
  return reinterpret_cast<uintptr_t>(p);
}
void symm_free(uintptr_t p) { TFT_CUDA_CHECK(cudaFree(P<void>(p))); }

// Base address + size of the cudaMalloc allocation containing `ptr` (so tensors
// living inside torch's caching-allocator segments can be exported over IPC).
py::tuple address_range(uintptr_t ptr) {
  typedef CUresult (*fn_t)(CUdeviceptr*, size_t*, CUdeviceptr);
  static fn_t fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    TFT_CUDA_CHECK(cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q));
    if (!f) throw std::runtime_error("cuMemGetAddressRange unavailable");
    fn = reinterpret_cast<fn_t>(f);
  }
  CUdeviceptr base = 0;
  size_t size = 0;
  CUresult r = fn(&base, &size, (CUdeviceptr)ptr);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuMemGetAddressRange failed: " + std::to_string((int)r));
  return py::make_tuple((uintptr_t)base, size);
}

// Whether cudaIpcGetMemHandle can export the allocation containing `ptr`. It cannot for cuMemCreate memory (vmm-mode
// symmetric segments, PyTorch's expandable segments); asking the driver first keeps a refused export from leaving an
// error behind for the next launch check.
bool ipc_capable(uintptr_t ptr) {
  typedef CUresult (*fn_t)(void*, CUpointer_attribute, CUdeviceptr);
  static fn_t fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    TFT_CUDA_CHECK(cudaGetDriverEntryPoint("cuPointerGetAttribute", &f, cudaEnableDefault, &q));
    if (!f) throw std::runtime_error("cuPointerGetAttribute unavailable");
    fn = reinterpret_cast<fn_t>(f);
  }
  int v = 0;
  CUresult r = fn(&v, CU_POINTER_ATTRIBUTE_IS_LEGACY_CUDA_IPC_CAPABLE, (CUdeviceptr)ptr);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuPointerGetAttribute failed: " + std::to_string((int)r));
  return v != 0;
}

void memset_async(uintptr_t p, int value, size_t nbytes, uintptr_t stream) {
  TFT_CUDA_CHECK(cudaMemsetAsync(P<void>(p), value, nbytes, S(stream)));
}
void memcpy_async(uintptr_t dst, uintptr_t src, size_t nbytes, uintptr_t stream) {
  TFT_CUDA_CHECK(cudaMemcpyAsync(P<void>(dst), P<void>(src), nbytes, cudaMemcpyDefault, S(stream)));
}
void memcpy_h2d(uintptr_t dst, const std::string& src, uintptr_t stream) {
  TFT_CUDA_CHECK(cudaMemcpyAsync(P<void>(dst), src.data(), src.size(), cudaMemcpyHostToDevice, S(stream)));
  TFT_CUDA_CHECK(cudaStreamSynchronize(S(stream)));
}
bool can_access_peer(int dev, int peer) {
  int ok = 0;
  TFT_CUDA_CHECK(cudaDeviceCanAccessPeer(&ok, dev, peer));
  return ok != 0;
}

}  // namespace

void bind_vmm(py::module_& m);  // vmm.cu

PYBIND11_MODULE(_K, m) {
  m.doc() = "torchft_b200 data-plane kernels (sm_90a): P2P all-reduce, q8 all-reduce, heal copy, model ops";
  m.attr("MAX_RANKS") = kMaxRanks;
  m.attr("MAX_BLOCKS") = kMaxBlocks;
  m.attr("NUM_SMS") = kNumSMs;
  m.attr("SIGNAL_CHANNELS") = kSignalChannels;
  m.attr("SIGNAL_PAD_BYTES") = sizeof(SignalPad);
  m.attr("Q8_GROUP") = 512;
  m.attr("ZERO1_MAX_NO_DECAY") = kMaxNoDecay;
  m.attr("ZERO1_MAX_BLOCKS") = kZero1MaxBlocks;
  m.attr("ZERO1_TOKSLOT_BYTES") = (int)sizeof(zero1::TokSlot);
  m.attr("ZERO1_VETO_ROWS") = zero1::kVetoRows;
  m.attr("ZERO1_BF16_MOMENTS") = true;  // zero1_update takes moment_dtype = bf16
  m.attr("ZERO1_EMA") = true;           // zero1_update takes an EMA of the weights and mode 2

  py::class_<Status>(m, "Status")
      .def(py::init<>())
      .def("dev_ptr", &Status::dev_ptr)
      .def("set_abort", &Status::set_abort)
      .def("aborted", &Status::aborted)
      .def("error", &Status::error)
      .def("clear", &Status::clear)
      .def("verdict", &Status::verdict)
      .def("grad_norm", &Status::grad_norm)
      .def("reason", &Status::reason)
      .def("set_timeout_ms", &Status::set_timeout_ms)
      .def("timeout_ms", &Status::timeout_ms);

  py::class_<MappedWords>(m, "MappedWords")
      .def(py::init<size_t>())
      .def("dev_ptr", &MappedWords::dev_ptr)
      .def("size", &MappedWords::size)
      .def("read", &MappedWords::read);

  py::class_<PeerTableH>(m, "PeerTable")
      .def(py::init<const std::vector<uintptr_t>&, const std::vector<uintptr_t>&, int, int>(),
           py::arg("data"), py::arg("pads"), py::arg("rank"), py::arg("world"))
      .def("with_data", &PeerTableH::with_data)
      .def("set_timeout_ms", &PeerTableH::set_timeout_ms)
      .def_property_readonly("rank", &PeerTableH::rank)
      .def_property_readonly("world", &PeerTableH::world);

  m.def("symm_alloc", &symm_alloc);
  m.def("symm_free", &symm_free);
  m.def("ipc_get_handle", &ipc_get_handle);
  m.def("ipc_open_handle", &ipc_open_handle);
  m.def("ipc_close_handle", &ipc_close_handle);
  m.def("address_range", &address_range);
  m.def("ipc_capable", &ipc_capable);
  m.def("memset_async", &memset_async);
  m.def("memcpy_async", &memcpy_async);
  m.def("memcpy_h2d", &memcpy_h2d);
  m.def("can_access_peer", &can_access_peer);

  m.def(
      "allreduce",
      [](const PeerTableH& pt, const Status& st, size_t off, uintptr_t user_in, uintptr_t user_out,
         size_t nelem, int dtype, int op, float scale, uint64_t flag, int channel, bool contribute,
         int algo, int blocks, int threads, uintptr_t stream) {
        allreduce_launch(pt.pt, st.dev(), off, P<void>(user_in), P<void>(user_out), nelem, dtype, op,
                         scale, flag, channel, contribute ? 1 : 0, algo, blocks, threads, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("off"), py::arg("user_in"), py::arg("user_out"),
      py::arg("nelem"), py::arg("dtype"), py::arg("op"), py::arg("scale"), py::arg("flag"),
      py::arg("channel"), py::arg("contribute"), py::arg("algo"), py::arg("blocks"),
      py::arg("threads"), py::arg("stream"));

  bind_vmm(m);
  m.def(
      "allreduce_nvls",
      [](const PeerTableH& pt, const Status& st, uintptr_t mc_base, size_t off, size_t nelem, int dtype, float scale,
         uint64_t flag, int channel, bool contribute, int blocks, int threads, uintptr_t stream) {
        allreduce_nvls_launch(pt.pt, st.dev(), P<void>(mc_base), off, nelem, dtype, scale, flag, channel,
                              contribute ? 1 : 0, blocks, threads, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("mc_base"), py::arg("off"), py::arg("nelem"), py::arg("dtype"),
      py::arg("scale"), py::arg("flag"), py::arg("channel"), py::arg("contribute"), py::arg("blocks"),
      py::arg("threads"), py::arg("stream"));

  m.def(
      "zero1_handshake",
      [](const PeerTableH& pt, const Status& st, uintptr_t ok_out, uint64_t flag, int channel, bool release,
         uintptr_t stream) {
        zero1::HsArgs a{};
        a.pt = pt.pt;
        a.st = st.dev();
        a.ok_out = P<int>(ok_out);
        a.flag = flag;
        a.channel = channel;
        a.release = release;
        zero1_handshake_launch(a, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("ok_out"), py::arg("flag"), py::arg("channel"), py::arg("release"),
      py::arg("stream"));
  m.def(
      "zero1_reduce",
      [](const PeerTableH& pt, uintptr_t ok, uintptr_t mc_base, size_t off, size_t nelem, float scale, int replication,
         uintptr_t gn, uintptr_t cta_sq, uintptr_t ticket, uintptr_t acc, int acc_mode, int blocks, int threads,
         uintptr_t stream) {
        zero1::RSArgs a{};
        a.pt = pt.pt;
        a.ok = P<const int>(ok);
        a.mc = P<char>(mc_base);
        a.off = off;
        a.nelem = nelem;
        a.scale = scale;
        a.replication = replication;
        a.gn = P<double>(gn);
        a.cta_sq = P<double>(cta_sq);
        a.ticket = P<unsigned>(ticket);
        a.acc = P<float>(acc);
        zero1_reduce_launch(a, acc_mode, blocks, threads, S(stream));
      },
      py::arg("pt"), py::arg("ok"), py::arg("mc_base"), py::arg("off"), py::arg("nelem"), py::arg("scale"),
      py::arg("replication"), py::arg("gn"), py::arg("cta_sq"), py::arg("ticket"), py::arg("acc"), py::arg("acc_mode"),
      py::arg("blocks"), py::arg("threads"), py::arg("stream"));
  m.def(
      "zero1_commit",
      [](const PeerTableH& pt, const Status& st, uintptr_t gate, uint64_t flag, uint32_t seq, int channel, bool host_ok,
         bool exchange, const std::vector<uintptr_t>& gnorm, int nunits, float max_norm, uintptr_t norm,
         const std::vector<uintptr_t>& tm, uintptr_t n_src, uintptr_t loss_src, long long rows, long long pmc,
         bool contribute, uintptr_t tm_out, uintptr_t tm_count, uintptr_t stream) {
        if (!gnorm.empty() && (int)gnorm.size() != pt.pt.world)
          throw std::runtime_error("zero1_commit: need one z1_gnorm pointer per rank");
        if (!tm.empty() && (int)tm.size() != pt.pt.world)
          throw std::runtime_error("zero1_commit: need one z1_tokmean slot per rank");
        zero1::CommitArgs a{};
        a.pt = pt.pt;
        a.st = st.dev();
        a.gate = P<int>(gate);
        a.flag = flag;
        a.seq = seq;
        a.channel = channel;
        a.host_ok = host_ok;
        a.exchange = exchange;
        for (size_t r = 0; r < gnorm.size(); ++r) a.gn[r] = P<const double>(gnorm[r]);
        a.nunits = nunits;
        a.max_norm = max_norm;
        a.norm = P<float>(norm);
        for (size_t r = 0; r < tm.size(); ++r) a.tm[r] = P<zero1::TokSlot>(tm[r]);
        a.n_src = P<const long long>(n_src);
        a.loss_src = P<const double>(loss_src);
        a.rows = rows;
        a.pmc = pmc;
        a.contribute = contribute;
        a.tm_out = P<float>(tm_out);
        a.tm_count = P<long long>(tm_count);
        zero1_commit_launch(a, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("gate"), py::arg("flag"), py::arg("seq"), py::arg("channel"),
      py::arg("host_ok"), py::arg("exchange"), py::arg("gnorm"), py::arg("nunits"), py::arg("max_norm"), py::arg("norm"),
      py::arg("tm"), py::arg("n_src"), py::arg("loss_src"), py::arg("rows"), py::arg("pmc"), py::arg("contribute"),
      py::arg("tm_out"), py::arg("tm_count"), py::arg("stream"));
  m.def(
      "zero1_update",
      [](const PeerTableH& pt, uintptr_t mc_base, uintptr_t gate, size_t poff, uintptr_t grad, uintptr_t master, uintptr_t mm,
         uintptr_t v, size_t nelem, float lr, float b1, float b2, float eps, float wd, int replication, int mode,
         uintptr_t table, size_t soff, int page_shift, uintptr_t coef, uintptr_t lr_tab, int lr_steps,
         const std::vector<size_t>& no_decay, int moment_dtype, uintptr_t ema, float ema_c, int blocks, int threads,
         uintptr_t stream) {
        if (no_decay.size() & 1) throw std::runtime_error("zero1_update: no_decay is a flat list of (lo, hi) pairs");
        zero1::UpdArgs a{};
        a.pt = pt.pt;
        a.mc = P<char>(mc_base);
        a.gate = P<const int>(gate);
        a.poff = poff;
        a.grad = P<const __nv_bfloat16>(grad);
        a.master = P<float>(master);
        a.m = P<void>(mm);
        a.v = P<void>(v);
        a.nelem = nelem;
        a.lr = lr;
        a.b1 = b1;
        a.b2 = b2;
        a.eps = eps;
        a.wd = wd;
        a.replication = replication;
        a.mode = mode;
        a.table = P<const int>(table);
        a.soff = soff;
        a.page_shift = page_shift;
        a.coef = P<const float>(coef);
        a.lr_tab = P<const float>(lr_tab);
        a.lr_steps = lr_steps;
        a.n_nd = (int)(no_decay.size() / 2);
        for (int r = 0; r < std::min(a.n_nd, kMaxNoDecay); ++r) {  // the launcher rejects more
          a.nd_lo[r] = no_decay[2 * r];
          a.nd_hi[r] = no_decay[2 * r + 1];
        }
        a.ema = P<void>(ema);
        a.ema_c = ema_c;
        zero1_update_launch(a, moment_dtype, blocks, threads, S(stream));
      },
      py::arg("pt"), py::arg("mc_base"), py::arg("gate"), py::arg("poff"), py::arg("grad"), py::arg("master"),
      py::arg("m"), py::arg("v"), py::arg("nelem"), py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"),
      py::arg("wd"), py::arg("replication"), py::arg("mode"), py::arg("table"), py::arg("soff"), py::arg("page_shift"),
      py::arg("coef"), py::arg("lr_tab"), py::arg("lr_steps"), py::arg("no_decay"), py::arg("moment_dtype"),
      py::arg("ema"), py::arg("ema_c"), py::arg("blocks"), py::arg("threads"), py::arg("stream"));

  m.attr("Z1_DIGEST_CHUNK_WORDS") = audit::kDigestChunkWords;
  m.attr("Z1_AUDIT_REPORT_HEADER") = audit::kReportHeader;
  m.def(
      "z1_digest",
      [](uintptr_t table_dev, int nentries, size_t total_chunks, uintptr_t slots, int blocks, uintptr_t stream) {
        z1_digest_launch(P<void>(table_dev), nentries, total_chunks, P<unsigned long long>(slots), blocks, S(stream));
      },
      py::arg("table"), py::arg("nentries"), py::arg("total_chunks"), py::arg("slots"), py::arg("blocks"),
      py::arg("stream"));
  m.def(
      "z1_audit_compare",
      [](const PeerTableH& pt, const Status& st, uintptr_t ok, const MappedWords& report, uint64_t seq, int nunits,
         int stride, int k, int narrays, uintptr_t stream) {
        audit::CompareArgs a{};
        a.pt = pt.pt;
        a.st = st.dev();
        a.ok = P<const int>(ok);
        a.report = P<unsigned long long>(report.dev_ptr());
        a.seq = seq;
        a.nunits = nunits;
        a.stride = stride;
        a.k = k;
        a.narrays = narrays;
        if (report.size() < (size_t)audit::kReportHeader + (size_t)pt.pt.world * ((size_t)nunits * stride + 1))
          throw std::runtime_error("z1_audit_compare: the report is too small for this quorum's slots");
        z1_audit_compare_launch(a, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("ok"), py::arg("report"), py::arg("seq"), py::arg("nunits"),
      py::arg("stride"), py::arg("k"), py::arg("narrays"), py::arg("stream"));

  m.def(
      "push_exchange",
      [](const PeerTableH& pt, const Status& st, uintptr_t in, uintptr_t out, const std::vector<size_t>& send_off,
         const std::vector<size_t>& send_len, const std::vector<size_t>& recv_len, const std::vector<size_t>& out_off,
         size_t slot_stride, uint64_t flag, int channel, int blocks, uintptr_t stream) {
        const size_t w = (size_t)pt.pt.world;
        if (send_off.size() != w || send_len.size() != w || recv_len.size() != w || out_off.size() != w)
          throw std::runtime_error("push_exchange: need one entry per rank");
        push_exchange_launch(pt.pt, st.dev(), P<void>(in), P<void>(out), send_off.data(), send_len.data(), recv_len.data(),
                             out_off.data(), slot_stride, flag, channel, blocks, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("input"), py::arg("output"), py::arg("send_off"), py::arg("send_len"),
      py::arg("recv_len"), py::arg("out_off"), py::arg("slot_stride"), py::arg("flag"), py::arg("channel"),
      py::arg("blocks"), py::arg("stream"));
  m.def(
      "reduce_scatter",
      [](const PeerTableH& pt, const Status& st, size_t off, uintptr_t user_in, uintptr_t out, size_t n, int dtype, int op,
         float scale, uint64_t flag, int channel, int blocks, uintptr_t stream) {
        reduce_scatter_launch(pt.pt, st.dev(), off, P<void>(user_in), P<void>(out), n, dtype, op, scale, flag, channel,
                              blocks, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("off"), py::arg("user_in"), py::arg("out"), py::arg("n"), py::arg("dtype"),
      py::arg("op"), py::arg("scale"), py::arg("flag"), py::arg("channel"), py::arg("blocks"), py::arg("stream"));
  m.def(
      "p2p",
      [](const PeerTableH& pt, const Status& st, bool is_send, uintptr_t buf, size_t nbytes, int peer, size_t mailbox_off,
         size_t mailbox_bytes, uint64_t seq0, int channel, uintptr_t stream) {
        p2p_launch(pt.pt, st.dev(), is_send ? 1 : 0, P<void>(buf), nbytes, peer, mailbox_off, mailbox_bytes, seq0, channel,
                   S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("is_send"), py::arg("buf"), py::arg("nbytes"), py::arg("peer"),
      py::arg("mailbox_off"), py::arg("mailbox_bytes"), py::arg("seq0"), py::arg("channel"), py::arg("stream"));

  m.def("q8_ngroups", &q8_ngroups);
  m.def("q8_buffer_bytes", &q8_buffer_bytes);
  m.def("q8_quantize", [](uintptr_t a, uintptr_t b, size_t nelem, size_t ngroups, int dtype, uintptr_t qbuf,
                          uintptr_t stream) {
    q8_quantize_launch(P<void>(a), P<void>(b), nelem, ngroups, dtype, P<void>(qbuf), S(stream));
  });
  m.def("q8_dequantize", [](uintptr_t qbuf, size_t ngroups, uintptr_t out, size_t nelem, int dtype,
                            uintptr_t stream) {
    q8_dequantize_launch(P<void>(qbuf), ngroups, P<void>(out), nelem, dtype, S(stream));
  });
  m.def("q8_reduce", [](uintptr_t srcs_dev, int nsrc, int first, size_t ngroups, size_t g_lo, size_t g_hi,
                        float post_scale, uintptr_t dst, uintptr_t stream) {
    q8_reduce_launch(P<const void* const>(srcs_dev), nsrc, first, ngroups, g_lo, g_hi, post_scale, P<void>(dst),
                     S(stream));
  });
  m.def(
      "q8_allreduce",
      [](const PeerTableH& pt, const Status& st, size_t off, uintptr_t in_a, uintptr_t in_b,
         uintptr_t out, size_t nelem, int dtype, float post_scale, uint64_t flag, int channel,
         bool contribute, int blocks, uintptr_t stream) {
        q8_allreduce_launch(pt.pt, st.dev(), off, P<void>(in_a), P<void>(in_b), P<void>(out), nelem,
                            dtype, post_scale, flag, channel, contribute ? 1 : 0, blocks, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("off"), py::arg("in_a"), py::arg("in_b"),
      py::arg("out"), py::arg("nelem"), py::arg("dtype"), py::arg("post_scale"), py::arg("flag"),
      py::arg("channel"), py::arg("contribute"), py::arg("blocks"), py::arg("stream"));

  m.def("q8_slice_buffer_bytes", &q8_slice_buffer_bytes);
  m.def("q8_slice_reduce", [](const PeerTableH& pt, uintptr_t ok, size_t q_off, size_t r_off, size_t nelem, float post_scale,
                               int blocks, uintptr_t stream) {
    q8_slice_reduce_launch(pt.pt, P<const int>(ok), q_off, r_off, nelem, post_scale, blocks, S(stream));
  });
  m.def("q8_gather_dequant", [](const PeerTableH& pt, uintptr_t ok, size_t r_off, size_t nelem, int dtype, uintptr_t out,
                                 int blocks, uintptr_t stream) {
    q8_gather_dequant_launch(pt.pt, P<const int>(ok), r_off, nelem, dtype, P<void>(out), blocks, S(stream));
  });
  m.def("q8_rs_buffer_bytes", &q8_rs_buffer_bytes);
  m.def(
      "q8_reduce_scatter",
      [](const PeerTableH& pt, const Status& st, size_t off, uintptr_t in, uintptr_t out, size_t nelem, size_t slice_elems,
         int dtype, float post_scale, uint64_t flag, int channel, bool contribute, int blocks, uintptr_t stream) {
        q8_reduce_scatter_launch(pt.pt, st.dev(), off, P<void>(in), P<void>(out), nelem, slice_elems, dtype, post_scale, flag,
                                 channel, contribute ? 1 : 0, blocks, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("off"), py::arg("input"), py::arg("out"), py::arg("nelem"),
      py::arg("slice_elems"), py::arg("dtype"), py::arg("post_scale"), py::arg("flag"), py::arg("channel"),
      py::arg("contribute"), py::arg("blocks"), py::arg("stream"));

  m.def("rmsnorm_fwd", [](uintptr_t x, uintptr_t w, uintptr_t y, uintptr_t rstd, int rows, int H,
                          float eps, uintptr_t s) {
    rmsnorm_fwd_launch(P<void>(x), P<void>(w), P<void>(y), P<float>(rstd), rows, H, eps, S(s));
  });
  m.def("rmsnorm_fwd_fp8", [](uintptr_t x, uintptr_t w, uintptr_t y8, uintptr_t yscale, uintptr_t rstd, int rows, int H,
                              float eps, uintptr_t s) {
    rmsnorm_fwd_fp8_launch(P<void>(x), P<void>(w), P<void>(y8), P<float>(yscale), P<float>(rstd), rows, H, eps, S(s));
  }, py::arg("x"), py::arg("w"), py::arg("y8"), py::arg("yscale"), py::arg("rstd"), py::arg("rows"), py::arg("H"),
     py::arg("eps"), py::arg("stream"));
  m.def("rmsnorm_bwd_grid", &rmsnorm_bwd_grid);
  m.def("rmsnorm_bwd", [](uintptr_t dy, uintptr_t x, uintptr_t w, uintptr_t rstd, uintptr_t dx,
                          uintptr_t dw_partial, uintptr_t dw, bool accumulate, int rows, int H,
                          uintptr_t s, uintptr_t dres) {
    rmsnorm_bwd_launch(P<void>(dy), P<void>(x), P<void>(w), P<float>(rstd), P<void>(dx),
                       P<float>(dw_partial), P<void>(dw), accumulate ? 1 : 0, rows, H, S(s), P<void>(dres));
  }, py::arg("dy"), py::arg("x"), py::arg("w"), py::arg("rstd"), py::arg("dx"), py::arg("dw_partial"),
     py::arg("dw"), py::arg("accumulate"), py::arg("rows"), py::arg("H"), py::arg("stream"), py::arg("dres") = 0);
  m.def("swiglu_fwd", [](uintptr_t gu, uintptr_t y, size_t T, int F, uintptr_t s) {
    swiglu_fwd_launch(P<void>(gu), P<void>(y), T, F, S(s));
  });
  m.def("swiglu_bwd", [](uintptr_t dy, uintptr_t gu, uintptr_t dgu, size_t T, int F, uintptr_t s) {
    swiglu_bwd_launch(P<void>(dy), P<void>(gu), P<void>(dgu), T, F, S(s));
  });
  m.def("rope_qkv", [](uintptr_t packed, size_t row, uintptr_t q, uintptr_t k, uintptr_t v, std::vector<int64_t> strides,
                       uintptr_t cs, size_t T, int S_, int D, int Hq, int Hkv, int dir, uintptr_t s, uintptr_t positions) {
    if (strides.size() != 9) throw std::runtime_error("rope_qkv: strides = (batch, position, head) x (q, k, v)");
    rope_qkv_launch(P<void>(packed), row, P<void>(q), P<void>(k), P<void>(v), strides.data(), P<void>(cs), T, S_, D, Hq,
                    Hkv, dir, S(s), P<const int>(positions));
  }, "RoPE + q/k/v split of a packed projection (dir 0) or its backward (dir 1), one launch; positions (int32 [T], "
     "optional) rotates token t by positions[t] instead of its offset in its row",
     py::arg("packed"), py::arg("row"), py::arg("q"), py::arg("k"), py::arg("v"), py::arg("strides"), py::arg("cs"),
     py::arg("T"), py::arg("S"), py::arg("D"), py::arg("Hq"), py::arg("Hkv"), py::arg("dir"), py::arg("stream"),
     py::arg("positions") = 0);
  m.def("xent", [](uintptr_t logits, uintptr_t target, uintptr_t loss, size_t rows, int V,
                   size_t row_stride, float grad_scale, long long ignore_index, uintptr_t s, uintptr_t scale) {
    xent_launch(P<void>(logits), P<void>(target), P<float>(loss), rows, V, row_stride, grad_scale,
                ignore_index, S(s), P<const float>(scale));
  }, py::arg("logits"), py::arg("target"), py::arg("loss"), py::arg("rows"), py::arg("V"), py::arg("row_stride"),
     py::arg("grad_scale"), py::arg("ignore_index"), py::arg("stream"), py::arg("scale") = 0);
  m.def("embedding_bwd_pieces", &embedding_bwd_pieces, "rows of the embedding_bwd partial scratch [pieces, 2, d] for T tokens");
  m.def("embedding_bwd", [](uintptr_t sorted_ids, uintptr_t perm, uintptr_t dx, size_t ldx, uintptr_t grad,
                            uintptr_t partial, int T, int d, uintptr_t s) {
    embedding_bwd_launch(P<const int64_t>(sorted_ids), P<const int64_t>(perm), P<void>(dx), ldx, P<void>(grad),
                         P<float>(partial), T, d, S(s));
  }, "grad[v] += sum of the dx rows of the tokens with id v, in place (stably sorted ids and their token indices)",
     py::arg("sorted_ids"), py::arg("perm"), py::arg("dx"), py::arg("ldx"), py::arg("grad"), py::arg("partial"),
     py::arg("T"), py::arg("d"), py::arg("stream"));
  m.def("adamw", [](uintptr_t p, uintptr_t master, uintptr_t mm, uintptr_t v, uintptr_t g, size_t n,
                    float lr, float b1, float b2, float eps, float wd, float bc1, float bc2,
                    float gscale, uintptr_t gate, uintptr_t s, int max_blocks) {
    adamw_launch(P<void>(p), P<float>(master), P<float>(mm), P<float>(v), P<void>(g), n, lr, b1, b2,
                 eps, wd, bc1, bc2, gscale, P<const int>(gate), max_blocks, S(s));
  }, py::arg("p"), py::arg("master"), py::arg("m"), py::arg("v"), py::arg("g"), py::arg("n"), py::arg("lr"),
     py::arg("b1"), py::arg("b2"), py::arg("eps"), py::arg("wd"), py::arg("bc1"), py::arg("bc2"),
     py::arg("gscale"), py::arg("gate"), py::arg("stream"), py::arg("max_blocks") = 0);
  m.def("diloco_outer", [](uintptr_t param, uintptr_t original, uintptr_t grad, uintptr_t mom, size_t n, int dtype, float lr,
                            float mu, bool nesterov, float alpha, uintptr_t gate, uintptr_t s) {
    diloco_outer_launch(P<void>(param), P<void>(original), P<void>(grad), P<float>(mom), n, dtype, lr, mu, nesterov ? 1 : 0,
                        alpha, P<const int>(gate), S(s));
  }, py::arg("param"), py::arg("original"), py::arg("grad"), py::arg("mom"), py::arg("n"), py::arg("dtype"), py::arg("lr"),
     py::arg("mu"), py::arg("nesterov"), py::arg("alpha"), py::arg("gate"), py::arg("stream"));
  m.def("fp8_rows", [](uintptr_t x, size_t ld, uintptr_t q, uintptr_t scale, int rows, int C, uintptr_t s) {
    fp8_rows_launch(P<void>(x), ld, P<void>(q), P<float>(scale), rows, C, S(s));
  }, py::arg("x"), py::arg("ld"), py::arg("q"), py::arg("scale"), py::arg("rows"), py::arg("C"), py::arg("stream"));
  m.def("fp8_rows_shape", &fp8_rows_shape, "(chunks per thread, threads) of the fp8_rows / fp8_swiglu CTA for a row of C");
  m.def("fp8_swiglu", [](uintptr_t gu, uintptr_t q, uintptr_t scale, int T, int F, uintptr_t s) {
    fp8_swiglu_launch(P<void>(gu), P<void>(q), P<float>(scale), T, F, S(s));
  }, py::arg("gu"), py::arg("q"), py::arg("scale"), py::arg("T"), py::arg("F"), py::arg("stream"));
  m.def("fp8_cols_t", [](uintptr_t w, int N, int K, uintptr_t q, uintptr_t scale, uintptr_t amax_ws, uintptr_t s) {
    fp8_cols_t_launch(P<void>(w), N, K, P<void>(q), P<float>(scale), P<uint32_t>(amax_ws), S(s));
  }, py::arg("w"), py::arg("N"), py::arg("K"), py::arg("q"), py::arg("scale"), py::arg("amax_ws"), py::arg("stream"));
  m.def("heal_copy", [](uintptr_t table_dev, int nentries, size_t total_chunks, size_t chunk_bytes,
                        int blocks, uintptr_t s) {
    heal_copy_launch(P<void>(table_dev), nentries, total_chunks, chunk_bytes, blocks, S(s));
  });
}
