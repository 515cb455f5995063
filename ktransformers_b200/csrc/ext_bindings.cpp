// pybind11 module `kt_kernel_ext_b200`: the reference's native extension surface for this path, bound to libktb200.so.
//
// Mirrors kt-kernel/ext_bindings.cpp (`kt_kernel_ext`):
//   moe.MOEConfig(expert_num, routed_expert_num, hidden_size, intermediate_size[, gpu_experts_mask_ptr]) + rw fields   (:746-831)
//   bind_moe_module<T>(m, name): __init__(MOEConfig), warm_up_task(), load_weights_task([physical_to_logical_map]),
//       forward_task(qlen_ptr, k, expert_ids, weights, input, output[, incremental]) -> (fn_ptr, args_ptr),
//       warm_up(), load_weights(), forward(...)                                                                          (:447-471)
//   CPUInfer(thread_num).submit / sync / submit_with_cuda_stream / sync_with_cuda_stream                                 (:554-565)
// Same task protocol: a task is the pair (function pointer, heap-allocated Args*); `submit` stores itself into
// Args::cpuinfer and calls the function (the reference leaks Args the same way, :193, :243).  What differs is WHERE the work
// runs: the reference enqueues onto CPU worker threads and orders them against a CUDA stream with host functions; here every
// task is a stream-ordered kernel launch, so `submit_with_cuda_stream(stream, task)` launches on `stream`, `submit(task)` on
// the CPUInfer's own stream (default: the legacy stream), and the `sync*` calls wait for / order against that stream.
// expert_ids / weights / input / output are DEVICE pointers (the experts are HBM-resident); qlen_ptr is a HOST int* read when
// the task runs, like the reference's `int qlen = *qlen_ptr` (kt-kernel/operators/moe-tp.hpp:209).
// Errors: a failing call throws std::runtime_error with ktb200_last_error() (reference: exceptions -> Python, :88-92).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>

#include "../../include/ktb200.h"

namespace py = pybind11;

static void check(int rc, const char* what) {
    if (rc != KTB200_OK) throw std::runtime_error(std::string(what) + ": " + ktb200_last_error());
}

struct GeneralMOEConfig {   // field names of kt-kernel/operators/common.hpp GeneralMOEConfig
    int expert_num = 0, num_experts_per_tok = 0, hidden_size = 0, intermediate_size = 0, layer_idx = 0;
    int max_len = 0, group_min_len = 10, group_max_len = 1024, m_block = 32;
    int gate_type = KTB200_TYPE_Q4_K, up_type = KTB200_TYPE_Q4_K, down_type = KTB200_TYPE_Q6_K, hidden_type = KTB200_TYPE_BF16;
    void *gate_proj = nullptr, *up_proj = nullptr, *down_proj = nullptr;
    void* physical_to_logical_map = nullptr;
    uint8_t* gpu_experts_mask = nullptr;
    int num_gpu_experts = 0;
    uintptr_t pool = 0;            // accepted for source compatibility (the reference's worker pool handle)
    int device = 0;                // CUDA device of the weight tensors
    int expert_id_offset = 0;      // expert-parallel shard: global id of local expert 0
    GeneralMOEConfig() = default;
    GeneralMOEConfig(int e, int k, int h, int i) : expert_num(e), num_experts_per_tok(k), hidden_size(h), intermediate_size(i) {}
};

class CPUInfer {   // kt-kernel/cpu_backend/cpuinfer.h:39-119: here a stream-ordered launcher
   public:
    explicit CPUInfer(int /*thread_num*/) {}
    void* stream = nullptr;        // where `submit` launches; submit_with_cuda_stream overrides it per task
    uintptr_t backend_ = 0;
    void submit(std::pair<intptr_t, intptr_t> task) { run(task, stream); }
    void submit_with_cuda_stream(intptr_t user_cuda_stream, std::pair<intptr_t, intptr_t> task) { run(task, (void*)user_cuda_stream); }
    void sync(int /*allow_n_pending*/ = 0) {
        if (cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) throw std::runtime_error("CPUInfer.sync: CUDA error");
    }
    void sync_with_cuda_stream(intptr_t /*user_cuda_stream*/, int /*allow_n_pending*/ = 0) {}   // already ordered on that stream
    void* current = nullptr;       // stream of the task being submitted (read by the task bodies)
   private:
    void run(std::pair<intptr_t, intptr_t> task, void* s) {
        current = s;
        void (*fn)(void*) = (void (*)(void*))task.first;
        void* args = (void*)task.second;
        *(CPUInfer**)args = this;   // Args::cpuinfer is the first member, as in the reference
        fn(args);
    }
};

class B200_MOE {   // the T of bind_moe_module<T>: GGUF K-quant experts resident in HBM on the sm_90a kernels
   public:
    explicit B200_MOE(const GeneralMOEConfig& c) : config(c) {
        ktb200_moe_config k{};
        k.expert_num = c.expert_num; k.routed_expert_num = c.num_experts_per_tok; k.hidden_size = c.hidden_size;
        k.intermediate_size = c.intermediate_size; k.stride = c.m_block; k.group_min_len = c.group_min_len;
        k.group_max_len = c.max_len > 0 ? c.max_len : c.group_max_len; k.use_silu = 1;
        k.gate_proj = c.gate_proj; k.up_proj = c.up_proj; k.down_proj = c.down_proj;
        k.gate_type = c.gate_type; k.up_type = c.up_type; k.down_type = c.down_type; k.hidden_type = c.hidden_type;
        k.expert_id_offset = c.expert_id_offset;
        check(ktb200_moe_create(&k, c.device, &h), "MOE");
    }
    ~B200_MOE() { ktb200_moe_destroy(h); }
    B200_MOE(const B200_MOE&) = delete;
    void warm_up_on(void* s) { check(ktb200_moe_warm_up(h, s), "warm_up"); }
    void load_weights_on(void* s) { check(ktb200_moe_load_weights(h, s), "load_weights"); }
    void forward_on(intptr_t qlen_ptr, int k, intptr_t ids, intptr_t w, intptr_t in, intptr_t out, bool incremental, void* s) {
        if (incremental) throw std::runtime_error("forward: incremental accumulation is a CPU-side feature of the reference's NUMA merge; not supported");
        const int qlen = *(const int*)qlen_ptr;
        check(ktb200_moe_forward(h, qlen, k, (const int64_t*)ids, (const float*)w, (const void*)in, (void*)out, nullptr, s), "forward");
    }
    void warm_up() { warm_up_on(nullptr); }
    void load_weights() { load_weights_on(nullptr); }
    void forward_binding(intptr_t qlen_ptr, int k, intptr_t ids, intptr_t w, intptr_t in, intptr_t out, bool incremental) {
        forward_on(qlen_ptr, k, ids, w, in, out, incremental, nullptr);
    }
    GeneralMOEConfig config;
    ktb200_moe* h = nullptr;
};

// (fn_ptr, args_ptr) tasks, kt-kernel/ext_bindings.cpp:180-259
struct WarmUpArgs { CPUInfer* cpuinfer; B200_MOE* moe; };
static void warm_up_inner(void* a) { auto* x = (WarmUpArgs*)a; x->moe->warm_up_on(x->cpuinfer->current); }
struct LoadArgs { CPUInfer* cpuinfer; B200_MOE* moe; };
static void load_inner(void* a) { auto* x = (LoadArgs*)a; x->moe->load_weights_on(x->cpuinfer->current); }
struct ForwardArgs { CPUInfer* cpuinfer; B200_MOE* moe; intptr_t qlen; int k; intptr_t expert_ids, weights, input, output; bool incremental; };
static void forward_inner(void* a) {
    auto* x = (ForwardArgs*)a;
    x->moe->forward_on(x->qlen, x->k, x->expert_ids, x->weights, x->input, x->output, x->incremental, x->cpuinfer->current);
}

#define DEF_PTR_PROPERTY(cls, name)                                                        \
    def_property(                                                                          \
        #name, [](const cls& self) { return reinterpret_cast<uintptr_t>(self.name); },     \
        [](cls& self, uintptr_t val) { self.name = reinterpret_cast<void*>(val); })

PYBIND11_MODULE(kt_kernel_ext_b200, m) {
    m.doc() = "H100 (sm_90a) drop-in for kt_kernel_ext's MoE path";
    m.def("version", [] { return std::string(ktb200_version()); });
    py::class_<CPUInfer>(m, "CPUInfer")
        .def(py::init<int>())
        .def("submit", &CPUInfer::submit)
        .def("sync", &CPUInfer::sync, py::arg("allow_n_pending") = 0)
        .def_readwrite("backend_", &CPUInfer::backend_)
        .def_property("stream", [](const CPUInfer& s) { return (uintptr_t)s.stream; }, [](CPUInfer& s, uintptr_t v) { s.stream = (void*)v; })
        .def("sync_with_cuda_stream", &CPUInfer::sync_with_cuda_stream, py::arg("user_cuda_stream"), py::arg("allow_n_pending") = 0)
        .def("submit_with_cuda_stream", &CPUInfer::submit_with_cuda_stream);

    auto moe_module = m.def_submodule("moe");
    py::class_<GeneralMOEConfig>(moe_module, "MOEConfig")
        .def(py::init([](int e, int k, int h, int i) { return GeneralMOEConfig(e, k, h, i); }))
        .def(py::init([](int e, int k, int h, int i, uintptr_t mask) {
            GeneralMOEConfig c(e, k, h, i);
            c.gpu_experts_mask = reinterpret_cast<uint8_t*>(mask);
            return c;
        }))
        .def_readwrite("expert_num", &GeneralMOEConfig::expert_num)
        .def_readwrite("num_experts_per_tok", &GeneralMOEConfig::num_experts_per_tok)
        .def_readwrite("hidden_size", &GeneralMOEConfig::hidden_size)
        .def_readwrite("intermediate_size", &GeneralMOEConfig::intermediate_size)
        .def_readwrite("layer_idx", &GeneralMOEConfig::layer_idx)
        .def_readwrite("pool", &GeneralMOEConfig::pool)
        .def_readonly("num_gpu_experts", &GeneralMOEConfig::num_gpu_experts)
        .def_property(
            "gpu_experts_mask", [](const GeneralMOEConfig& s) { return reinterpret_cast<uintptr_t>(s.gpu_experts_mask); },
            [](GeneralMOEConfig& s, uintptr_t v) { s.gpu_experts_mask = reinterpret_cast<uint8_t*>(v); })
        .DEF_PTR_PROPERTY(GeneralMOEConfig, physical_to_logical_map)
        .DEF_PTR_PROPERTY(GeneralMOEConfig, gate_proj)
        .DEF_PTR_PROPERTY(GeneralMOEConfig, up_proj)
        .DEF_PTR_PROPERTY(GeneralMOEConfig, down_proj)
        .def_readwrite("max_len", &GeneralMOEConfig::max_len)
        .def_readwrite("m_block", &GeneralMOEConfig::m_block)
        .def_readwrite("group_min_len", &GeneralMOEConfig::group_min_len)
        .def_readwrite("group_max_len", &GeneralMOEConfig::group_max_len)
        .def_readwrite("gate_type", &GeneralMOEConfig::gate_type)
        .def_readwrite("up_type", &GeneralMOEConfig::up_type)
        .def_readwrite("down_type", &GeneralMOEConfig::down_type)
        .def_readwrite("hidden_type", &GeneralMOEConfig::hidden_type)
        .def_readwrite("device", &GeneralMOEConfig::device)
        .def_readwrite("expert_id_offset", &GeneralMOEConfig::expert_id_offset);

    // bind_moe_module<B200_MOE>(moe_module, "B200_MOE")
    py::class_<B200_MOE, std::shared_ptr<B200_MOE>>(moe_module, "B200_MOE")
        .def(py::init<GeneralMOEConfig>())
        .def("warm_up_task", [](std::shared_ptr<B200_MOE> moe) {
            return std::make_pair((intptr_t)&warm_up_inner, (intptr_t) new WarmUpArgs{nullptr, moe.get()});
        })
        .def("load_weights_task", [](std::shared_ptr<B200_MOE> moe) {
            return std::make_pair((intptr_t)&load_inner, (intptr_t) new LoadArgs{nullptr, moe.get()});
        })
        .def("load_weights_task", [](std::shared_ptr<B200_MOE> moe, uintptr_t physical_to_logical_map) {
            if (physical_to_logical_map) moe->config.physical_to_logical_map = reinterpret_cast<void*>(physical_to_logical_map);
            return std::make_pair((intptr_t)&load_inner, (intptr_t) new LoadArgs{nullptr, moe.get()});
        }, py::arg("physical_to_logical_map"))
        .def("forward_task", [](std::shared_ptr<B200_MOE> moe, intptr_t qlen, int k, intptr_t ids, intptr_t w, intptr_t in, intptr_t out) {
            return std::make_pair((intptr_t)&forward_inner, (intptr_t) new ForwardArgs{nullptr, moe.get(), qlen, k, ids, w, in, out, false});
        })
        .def("forward_task", [](std::shared_ptr<B200_MOE> moe, intptr_t qlen, int k, intptr_t ids, intptr_t w, intptr_t in, intptr_t out, bool inc) {
            return std::make_pair((intptr_t)&forward_inner, (intptr_t) new ForwardArgs{nullptr, moe.get(), qlen, k, ids, w, in, out, inc});
        })
        .def("warm_up", &B200_MOE::warm_up)
        .def("load_weights", &B200_MOE::load_weights)
        .def("forward", &B200_MOE::forward_binding);
}
