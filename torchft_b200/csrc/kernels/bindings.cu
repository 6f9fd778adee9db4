// pybind11 surface of the data-plane extension `torchft_b200._K`.
//
// Design: Python owns policy (which buffers, which peers, which stream); this
// module owns mechanism (peer-memory handles, status block, kernel launches).
// All pointers/streams cross the boundary as integers, so there is no torch
// ABI dependency and the module imports on a CPU-only box (calls then raise).
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "api.h"
#include "common.cuh"

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
  void set_timeout_ms(double ms) { host_->timeout_ns = (uint64_t)(ms * 1e6); }
  double timeout_ms() const { return (double)host_->timeout_ns / 1e6; }
  StatusBlock* dev() const { return dev_; }

 private:
  StatusBlock* host_ = nullptr;
  StatusBlock* dev_ = nullptr;
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

  py::class_<Status>(m, "Status")
      .def(py::init<>())
      .def("dev_ptr", &Status::dev_ptr)
      .def("set_abort", &Status::set_abort)
      .def("aborted", &Status::aborted)
      .def("error", &Status::error)
      .def("clear", &Status::clear)
      .def("verdict", &Status::verdict)
      .def("set_timeout_ms", &Status::set_timeout_ms)
      .def("timeout_ms", &Status::timeout_ms);

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
  m.def("memset_async", &memset_async);
  m.def("memcpy_async", &memcpy_async);
  m.def("memcpy_h2d", &memcpy_h2d);
  m.def("can_access_peer", &can_access_peer);

  m.def(
      "allreduce",
      [](const PeerTableH& pt, const Status& st, size_t off, uintptr_t user_in, uintptr_t user_out,
         size_t nelem, int dtype, int op, float scale, uint64_t flag, int channel, bool contribute,
         int algo, int blocks, int threads, int barrier_mode, uintptr_t stream) {
        allreduce_launch(pt.pt, st.dev(), off, P<void>(user_in), P<void>(user_out), nelem, dtype, op,
                         scale, flag, channel, contribute ? 1 : 0, algo, blocks, threads, barrier_mode, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("off"), py::arg("user_in"), py::arg("user_out"),
      py::arg("nelem"), py::arg("dtype"), py::arg("op"), py::arg("scale"), py::arg("flag"),
      py::arg("channel"), py::arg("contribute"), py::arg("algo"), py::arg("blocks"),
      py::arg("threads"), py::arg("barrier_mode"), py::arg("stream"));

  bind_vmm(m);
  m.def(
      "allreduce_nvls",
      [](const PeerTableH& pt, const Status& st, uintptr_t mc_base, size_t off, size_t nelem, int dtype, float scale,
         uint64_t flag, int channel, bool contribute, int blocks, int threads, int barrier_mode, uintptr_t stream) {
        allreduce_nvls_launch(pt.pt, st.dev(), P<void>(mc_base), off, nelem, dtype, scale, flag, channel,
                              contribute ? 1 : 0, blocks, threads, barrier_mode, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("mc_base"), py::arg("off"), py::arg("nelem"), py::arg("dtype"),
      py::arg("scale"), py::arg("flag"), py::arg("channel"), py::arg("contribute"), py::arg("blocks"),
      py::arg("threads"), py::arg("barrier_mode"), py::arg("stream"));

  m.def(
      "zero1_handshake",
      [](const PeerTableH& pt, const Status& st, uintptr_t ok_out, uint64_t flag, int channel, bool release, int barrier_mode,
         uintptr_t stream) {
        zero1_handshake_launch(pt.pt, st.dev(), P<int>(ok_out), flag, channel, release ? 1 : 0, barrier_mode, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("ok_out"), py::arg("flag"), py::arg("channel"), py::arg("release"),
      py::arg("barrier_mode"), py::arg("stream"));
  m.def(
      "zero1_reduce",
      [](const PeerTableH& pt, uintptr_t ok, uintptr_t mc_base, size_t off, size_t nelem, float scale, int replication,
         int blocks, int threads, uintptr_t stream) {
        zero1_reduce_launch(pt.pt, P<const int>(ok), P<void>(mc_base), off, nelem, scale, replication, blocks, threads, S(stream));
      },
      py::arg("pt"), py::arg("ok"), py::arg("mc_base"), py::arg("off"), py::arg("nelem"), py::arg("scale"),
      py::arg("replication"), py::arg("blocks"), py::arg("threads"), py::arg("stream"));
  m.def(
      "zero1_commit",
      [](const PeerTableH& pt, const Status& st, uintptr_t gate, uint64_t flag, uint32_t seq, int channel,
         bool host_ok, bool exchange, uintptr_t stream) {
        zero1_commit_launch(pt.pt, st.dev(), P<int>(gate), flag, seq, channel, host_ok ? 1 : 0, exchange ? 1 : 0,
                            S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("gate"), py::arg("flag"), py::arg("seq"), py::arg("channel"),
      py::arg("host_ok"), py::arg("exchange"), py::arg("stream"));
  m.def(
      "zero1_update",
      [](const PeerTableH& pt, uintptr_t mc_base, uintptr_t gate, size_t poff, uintptr_t grad, uintptr_t master, uintptr_t mm,
         uintptr_t v, size_t nelem, float lr, float b1, float b2, float eps, float wd, int replication, int mode,
         int blocks, int threads, uintptr_t stream) {
        zero1_update_launch(pt.pt, P<void>(mc_base), P<const int>(gate), poff, P<void>(grad), P<float>(master), P<float>(mm),
                            P<float>(v), nelem, lr, b1, b2, eps, wd, replication, mode, blocks, threads, S(stream));
      },
      py::arg("pt"), py::arg("mc_base"), py::arg("gate"), py::arg("poff"), py::arg("grad"), py::arg("master"),
      py::arg("m"), py::arg("v"), py::arg("nelem"), py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"),
      py::arg("wd"), py::arg("replication"), py::arg("mode"), py::arg("blocks"), py::arg("threads"), py::arg("stream"));

  m.def(
      "push_exchange",
      [](const PeerTableH& pt, const Status& st, uintptr_t in, uintptr_t out, const std::vector<size_t>& send_off,
         const std::vector<size_t>& send_len, const std::vector<size_t>& recv_len, const std::vector<size_t>& out_off,
         size_t slot_stride, uint64_t flag, int channel, int blocks, int barrier_mode, uintptr_t stream) {
        const size_t w = (size_t)pt.pt.world;
        if (send_off.size() != w || send_len.size() != w || recv_len.size() != w || out_off.size() != w)
          throw std::runtime_error("push_exchange: need one entry per rank");
        push_exchange_launch(pt.pt, st.dev(), P<void>(in), P<void>(out), send_off.data(), send_len.data(), recv_len.data(),
                             out_off.data(), slot_stride, flag, channel, blocks, barrier_mode, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("input"), py::arg("output"), py::arg("send_off"), py::arg("send_len"),
      py::arg("recv_len"), py::arg("out_off"), py::arg("slot_stride"), py::arg("flag"), py::arg("channel"),
      py::arg("blocks"), py::arg("barrier_mode"), py::arg("stream"));
  m.def(
      "reduce_scatter",
      [](const PeerTableH& pt, const Status& st, size_t off, uintptr_t user_in, uintptr_t out, size_t n, int dtype, int op,
         float scale, uint64_t flag, int channel, int blocks, int barrier_mode, uintptr_t stream) {
        reduce_scatter_launch(pt.pt, st.dev(), off, P<void>(user_in), P<void>(out), n, dtype, op, scale, flag, channel,
                              blocks, barrier_mode, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("off"), py::arg("user_in"), py::arg("out"), py::arg("n"), py::arg("dtype"),
      py::arg("op"), py::arg("scale"), py::arg("flag"), py::arg("channel"), py::arg("blocks"), py::arg("barrier_mode"),
      py::arg("stream"));
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
  m.def("q8_quantize", [](uintptr_t a, uintptr_t b, size_t nelem, int dtype, int world, uintptr_t qbuf,
                          uintptr_t stream) {
    q8_quantize_launch(P<void>(a), P<void>(b), nelem, dtype, world, P<void>(qbuf), S(stream));
  });
  m.def("q8_dequantize", [](uintptr_t qbuf, size_t nelem, int dtype, int world, uintptr_t out,
                            uintptr_t stream) {
    q8_dequantize_launch(P<void>(qbuf), nelem, dtype, world, P<void>(out), S(stream));
  });
  m.def("q8_reduce", [](uintptr_t srcs_dev, int world, int rank, size_t nelem, float post_scale,
                        uintptr_t dst, uintptr_t stream) {
    q8_reduce_launch(P<const void* const>(srcs_dev), world, rank, nelem, post_scale, P<void>(dst),
                     S(stream));
  });
  m.def("q8_quantize_raw", [](uintptr_t a, uintptr_t b, size_t nelem, size_t ngroups, int dtype, uintptr_t qbuf,
                              uintptr_t stream) {
    q8_quantize_raw_launch(P<void>(a), P<void>(b), nelem, ngroups, dtype, P<void>(qbuf), S(stream));
  });
  m.def("q8_dequantize_raw", [](uintptr_t qbuf, size_t ngroups, uintptr_t out, size_t nelem, int dtype,
                                uintptr_t stream) {
    q8_dequantize_raw_launch(P<void>(qbuf), ngroups, P<void>(out), nelem, dtype, S(stream));
  });
  m.def("q8_reduce_raw", [](uintptr_t srcs_dev, int nsrc, int first, size_t ngroups, size_t g_lo, size_t g_hi,
                            float post_scale, uintptr_t dst, uintptr_t stream) {
    q8_reduce_raw_launch(P<const void* const>(srcs_dev), nsrc, first, ngroups, g_lo, g_hi, post_scale, P<void>(dst),
                         S(stream));
  });
  m.def(
      "q8_allreduce",
      [](const PeerTableH& pt, const Status& st, size_t off, uintptr_t in_a, uintptr_t in_b,
         uintptr_t out, size_t nelem, int dtype, float post_scale, uint64_t flag, int channel,
         bool contribute, int blocks, int barrier_mode, uintptr_t stream) {
        q8_allreduce_launch(pt.pt, st.dev(), off, P<void>(in_a), P<void>(in_b), P<void>(out), nelem,
                            dtype, post_scale, flag, channel, contribute ? 1 : 0, blocks, barrier_mode, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("off"), py::arg("in_a"), py::arg("in_b"),
      py::arg("out"), py::arg("nelem"), py::arg("dtype"), py::arg("post_scale"), py::arg("flag"),
      py::arg("channel"), py::arg("contribute"), py::arg("blocks"), py::arg("barrier_mode"), py::arg("stream"));

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
         int dtype, float post_scale, uint64_t flag, int channel, bool contribute, int blocks, int barrier_mode,
         uintptr_t stream) {
        q8_reduce_scatter_launch(pt.pt, st.dev(), off, P<void>(in), P<void>(out), nelem, slice_elems, dtype, post_scale, flag,
                                 channel, contribute ? 1 : 0, blocks, barrier_mode, S(stream));
      },
      py::arg("pt"), py::arg("status"), py::arg("off"), py::arg("input"), py::arg("out"), py::arg("nelem"),
      py::arg("slice_elems"), py::arg("dtype"), py::arg("post_scale"), py::arg("flag"), py::arg("channel"),
      py::arg("contribute"), py::arg("blocks"), py::arg("barrier_mode"), py::arg("stream"));

  m.def("rmsnorm_fwd", [](uintptr_t x, uintptr_t w, uintptr_t y, uintptr_t rstd, int rows, int H,
                          float eps, uintptr_t s) {
    rmsnorm_fwd_launch(P<void>(x), P<void>(w), P<void>(y), P<float>(rstd), rows, H, eps, S(s));
  });
  m.def("rmsnorm_bwd_grid", &rmsnorm_bwd_grid);
  m.def("rmsnorm_tune", &rmsnorm_tune, "(0 forward | 1 backward, CTA size 128/256/512, prefetch next row, CTAs/SM at 128 threads)");
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
  m.def("rope", [](uintptr_t in, uintptr_t out, uintptr_t cs, size_t T, int S_, int heads, int D,
                   size_t in_stride, size_t out_stride, float sign, uintptr_t s) {
    rope_launch(P<void>(in), P<void>(out), P<void>(cs), T, S_, heads, D, in_stride, out_stride, sign, S(s));
  });
  m.def("rope_qkv", [](uintptr_t packed, size_t row, uintptr_t q, uintptr_t k, uintptr_t v, std::vector<int64_t> strides,
                       uintptr_t cs, size_t T, int S_, int D, int Hq, int Hkv, int dir, uintptr_t s) {
    if (strides.size() != 9) throw std::runtime_error("rope_qkv: strides = (batch, position, head) x (q, k, v)");
    rope_qkv_launch(P<void>(packed), row, P<void>(q), P<void>(k), P<void>(v), strides.data(), P<void>(cs), T, S_, D, Hq,
                    Hkv, dir, S(s));
  }, "RoPE + q/k/v split of a packed projection (dir 0) or its backward (dir 1), one launch");
  m.def("xent", [](uintptr_t logits, uintptr_t target, uintptr_t loss, size_t rows, int V,
                   size_t row_stride, float grad_scale, long long ignore_index, uintptr_t s) {
    xent_launch(P<void>(logits), P<void>(target), P<float>(loss), rows, V, row_stride, grad_scale,
                ignore_index, S(s));
  });
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
  m.def("sumsq", [](uintptr_t g, size_t n, uintptr_t out, uintptr_t s) {
    sumsq_launch(P<void>(g), n, P<float>(out), S(s));
  });
  m.def("heal_copy_bulk", [](uintptr_t table_dev, int nentries, size_t total_chunks, size_t chunk_bytes, int blocks, uintptr_t s) {
    heal_copy_bulk_launch(P<void>(table_dev), nentries, total_chunks, chunk_bytes, blocks, S(s));
  });
  m.def("heal_copy", [](uintptr_t table_dev, int nentries, size_t total_chunks, size_t chunk_bytes,
                        int blocks, uintptr_t s) {
    heal_copy_launch(P<void>(table_dev), nentries, total_chunks, chunk_bytes, blocks, S(s));
  });
}
