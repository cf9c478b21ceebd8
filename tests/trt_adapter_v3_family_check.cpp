// trt_adapter_v3_family_check.cpp -- the yolov3 family's YoloLayer_TRT creators of include/trtx_plugins.h (one per driver:
// yolov3, yolov4, scaled-yolov4, yolov3-tiny, yolov3-spp), compiled against tests/mock_trt/NvInfer.h.
//   (no argument)  createPlugin with an empty field collection, the blob round trip through deserializePlugin, refused
//                  lengths and foreign blobs, and the generic creator's behaviour on the same blobs;
//   --dump         prints each creator's serialized blob in hex for tests/test_yolov3_family_cpu.py to compare with the
//                  Python mirror and the drivers' own yololayer.h;
//   --gpu          enqueues each driver's plugin (both adapters) and compares the output with the direct C call.
#include "trtx_plugins.h"

#include <cuda_runtime_api.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <vector>

#define CHECK(x)                                                                      \
    do {                                                                              \
        if (!(x)) {                                                                   \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #x); \
            std::exit(1);                                                             \
        }                                                                             \
    } while (0)

using namespace nvinfer1;
using namespace trtx;

static std::vector<unsigned char> blob_of(IPluginV2* p) {
    std::vector<unsigned char> b(p->getSerializationSize());
    p->serialize(b.data());
    return b;
}

template <class Traits>
static void check_host(const char* name, bool dump) {
    YoloV3FamilyCreatorT<Traits, true> cr;
    YoloV3FamilyCreatorT<Traits, false> cr_io;
    CHECK(std::strcmp(cr.getPluginName(), "YoloLayer_TRT") == 0 && std::strcmp(cr.getPluginVersion(), "1") == 0);
    CHECK(cr.getFieldNames()->nbFields == 0);
    PluginFieldCollection empty{0, nullptr};
    cr.setPluginNamespace("ns1");
    IPluginV2* p = cr.createPlugin("yololayer", &empty);
    CHECK(p != nullptr && std::strcmp(p->getPluginNamespace(), "ns1") == 0);
    CHECK(std::strcmp(p->getPluginType(), "YoloLayer_TRT") == 0);
    auto* dyn = dynamic_cast<YoloLayerPluginDynamic*>(p);
    CHECK(dyn != nullptr);
    const trtx_yolo_params& q = dyn->core().p;
    CHECK(q.variant == Traits::variant && q.num_classes == Traits::classes && q.max_out == Traits::max_out);
    CHECK(q.net_w == Traits::net_w && q.net_h == Traits::net_h && q.num_levels == Traits::levels && q.det_floats == 7);
    CHECK(dyn->core().out_elems() == 1 + Traits::max_out * 7);
    const int kb = Traits::variant == TRTX_YOLO_V3 ? 36 : 32;
    std::vector<unsigned char> b = blob_of(p);
    CHECK(b.size() == (size_t)(12 + kb * Traits::levels));
    IPluginV2* pn = cr.createPlugin("yololayer", nullptr);  // the reference never reads the collection
    CHECK(pn != nullptr && blob_of(pn) == b);
    pn->destroy();
    // the IOExt adapter gives the same blob
    IPluginV2* pio = cr_io.createPlugin("yololayer", &empty);
    CHECK(pio != nullptr && dynamic_cast<YoloLayerPluginIOExt*>(pio) != nullptr && blob_of(pio) == b);
    pio->destroy();
    // round trip
    IPluginV2* r = cr.deserializePlugin("yololayer", b.data(), b.size());
    CHECK(r != nullptr && blob_of(r) == b);
    CHECK(std::memcmp(&dynamic_cast<YoloLayerPluginDynamic*>(r)->core().p, &q, sizeof(q)) == 0);
    r->destroy();
    // a changed threadCount and anchor travel through the blob
    std::vector<unsigned char> b2 = b;
    const int tc = 64;
    const float a0 = 7.5f;
    std::memcpy(b2.data() + 4, &tc, 4);
    std::memcpy(b2.data() + 12 + kb - 24, &a0, 4);
    r = cr.deserializePlugin("yololayer", b2.data(), b2.size());
    CHECK(r != nullptr && blob_of(r) == b2);
    r->destroy();
    // malformed lengths and foreign layouts are refused
    std::vector<unsigned char> big(b.size() + 64, 0);
    std::memcpy(big.data(), b.data(), b.size());
    for (size_t len : {(size_t)0, (size_t)4, (size_t)11, (size_t)12, b.size() - 1, b.size() + 1, b.size() + 4, b.size() - 4,
                       b.size() + (size_t)kb, b.size() + (size_t)(68 - kb)})
        CHECK(cr.deserializePlugin("yololayer", big.data(), len) == nullptr);
    CHECK(cr.deserializePlugin("yololayer", nullptr, b.size()) == nullptr);
    std::vector<unsigned char> bk = b;  // kernelCount that does not match the length
    const int kc_bad = Traits::levels + 1;
    std::memcpy(bk.data() + 8, &kc_bad, 4);
    CHECK(cr.deserializePlugin("yololayer", bk.data(), bk.size()) == nullptr);
    // a 3-level yolov7 / YOLOP blob (24 + 32 * 3 = 120 bytes, spp's length at 3 levels) is refused by every family creator
    YoloCore v7;
    const int kernels7[3][8] = {{80, 80}, {40, 40}, {20, 20}};
    v7.init_v5(80, 640, 640, 1000, false, kernels7, 3, YoloCore::kV7Floats);
    std::vector<unsigned char> b7(v7.serial_size());
    v7.serialize(b7.data());
    CHECK(b7.size() == 120);
    CHECK(cr.deserializePlugin("yololayer", b7.data(), b7.size()) == nullptr);
    // the generic creator is unchanged: a family blob of 32-byte kernels is not one of its layouts, spp's 120 bytes
    // read as the yolov7 layout (the length cannot tell them apart)
    YoloPluginCreator gen;
    IPluginV2* g = gen.deserializePlugin("yololayer", b.data(), b.size());
    if (Traits::variant == TRTX_YOLO_V3) {
        CHECK(g != nullptr && dynamic_cast<YoloLayerPluginDynamic*>(g)->core().p.variant == TRTX_YOLO_V5);
        g->destroy();
    } else {
        CHECK(g == nullptr);
    }
    CHECK(gen.createPlugin("yololayer", &empty) == nullptr);
    if (dump) {
        std::printf("blob %s ", name);
        for (unsigned char c : b) std::printf("%02x", c);
        std::printf("\n");
    }
    p->destroy();
}

template <class Traits>
static void check_gpu(const char* name) {
    const int batch = 3;
    const int C = 3 * (5 + Traits::classes);
    YoloV3FamilyCreatorT<Traits, true> cr;
    YoloV3FamilyCreatorT<Traits, false> cr_io;
    PluginFieldCollection empty{0, nullptr};
    auto* dyn = static_cast<YoloLayerPluginDynamic*>(cr.createPlugin("yololayer", &empty));
    auto* io = static_cast<YoloLayerPluginIOExt*>(cr_io.createPlugin("yololayer", &empty));
    trtx_yolo_params q = dyn->core().p;
    std::mt19937 rng(17);
    std::normal_distribution<float> nd(-4.0f, 3.0f);
    std::vector<void*> in(Traits::levels);
    std::vector<PluginTensorDesc> desc(Traits::levels);
    for (int l = 0; l < Traits::levels; ++l) {
        const int gh = Traits::kernels()[l].h > 0 ? Traits::kernels()[l].h : 76 >> l;
        const int gw = Traits::kernels()[l].w > 0 ? Traits::kernels()[l].w : 76 >> l;
        q.grid_h[l] = gh;
        q.grid_w[l] = gw;
        std::vector<float> h((size_t)batch * C * gh * gw);
        for (auto& v : h) v = nd(rng);
        CHECK(cudaMalloc(&in[l], h.size() * 4) == cudaSuccess);
        CHECK(cudaMemcpy(in[l], h.data(), h.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess);
        desc[l].dims.nbDims = 4;
        desc[l].dims.d[0] = batch;
        desc[l].dims.d[1] = C;
        desc[l].dims.d[2] = gh;
        desc[l].dims.d[3] = gw;
        desc[l].type = DataType::kFLOAT;
        desc[l].format = TensorFormat::kLINEAR;
    }
    const size_t out_n = (size_t)batch * (1 + Traits::max_out * 7);
    const size_t ws_n = trtx_yolo_workspace_size(&q, batch);
    CHECK(ws_n > 0 && dyn->getWorkspaceSize(desc.data(), Traits::levels, nullptr, 1) >= ws_n);
    void *ws, *m_ref, *m_dyn, *m_io;
    CHECK(cudaMalloc(&m_ref, out_n * 4) == cudaSuccess && cudaMalloc(&m_dyn, out_n * 4) == cudaSuccess);
    CHECK(cudaMalloc(&m_io, out_n * 4) == cudaSuccess && cudaMalloc(&ws, ws_n) == cudaSuccess);
    float *o_ref = static_cast<float*>(m_ref), *o_dyn = static_cast<float*>(m_dyn), *o_io = static_cast<float*>(m_io);
    cudaMemset(o_ref, 0, out_n * 4);
    cudaMemset(o_dyn, 0, out_n * 4);
    cudaMemset(o_io, 0, out_n * 4);
    CHECK(trtx_yolo_decode_enqueue(&q, batch, in.data(), o_ref, ws, ws_n, nullptr) == 0);
    void* outs_dyn[1] = {o_dyn};
    CHECK(dyn->enqueue(desc.data(), nullptr, in.data(), outs_dyn, ws, nullptr) == 0);
    if (Traits::variant != TRTX_YOLO_V3) {  // spp's IOExt adapter has no grids (they come from the bound tensors)
        void* outs_io[1] = {o_io};
        CHECK(io->enqueue(batch, in.data(), outs_io, ws, nullptr) == 0);
    }
    CHECK(cudaDeviceSynchronize() == cudaSuccess);
    std::vector<float> a(out_n), b(out_n), c(out_n);
    cudaMemcpy(a.data(), o_ref, out_n * 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(b.data(), o_dyn, out_n * 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(c.data(), o_io, out_n * 4, cudaMemcpyDeviceToHost);
    CHECK(a[0] > 0 && std::memcmp(a.data(), b.data(), out_n * 4) == 0);
    if (Traits::variant != TRTX_YOLO_V3) CHECK(std::memcmp(a.data(), c.data(), out_n * 4) == 0);
    std::printf("%s gpu rows %d\n", name, (int)a[0]);
    for (void* p : in) cudaFree(p);
    cudaFree(o_ref);
    cudaFree(o_dyn);
    cudaFree(o_io);
    cudaFree(ws);
    dyn->destroy();
    io->destroy();
}

int main(int argc, char** argv) {
    const bool dump = argc > 1 && std::strcmp(argv[1], "--dump") == 0;
    const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
    check_host<YoloV3Traits>("yolov3", dump);
    check_host<YoloV4Traits>("yolov4", dump);
    check_host<ScaledYoloV4Traits>("scaled-yolov4", dump);
    check_host<YoloV3TinyTraits>("yolov3-tiny", dump);
    check_host<YoloV3SppTraits>("yolov3-spp", dump);
    std::printf("v3 family adapter check ok\n");
    if (gpu) {
        check_gpu<YoloV3Traits>("yolov3");
        check_gpu<YoloV4Traits>("yolov4");
        check_gpu<ScaledYoloV4Traits>("scaled-yolov4");
        check_gpu<YoloV3TinyTraits>("yolov3-tiny");
        check_gpu<YoloV3SppTraits>("yolov3-spp");
        std::printf("gpu enqueue ok\n");
    }
    return 0;
}
