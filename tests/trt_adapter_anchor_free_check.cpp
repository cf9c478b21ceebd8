// trt_adapter_anchor_free_check.cpp -- the YoloLayer_TRT creators of yolov9 (YoloV9PluginCreator) and yolov10 / yolov13
// (YoloV10PluginCreator) of include/trtx_plugins.h, compiled against tests/mock_trt/NvInfer.h.
//   (no argument)  registry lookup -> createPlugin -> serialize -> deserializePlugin on both adapters, refused field
//                  collections and blobs, and the generic creator's behaviour on the same fields and blobs;
//   --dump         prints the blobs of the drivers' own configurations in hex for tests/test_anchor_free_cpu.py to compare
//                  with the Python mirrors and the drivers' compiled plugins;
//   --gpu          also enqueues each plugin (both adapters) and compares the output with the direct C call.
#define TRTX_REGISTER_PLUGINS
#define TRTX_YOLO_ANCHOR_FREE 9
#include "trtx_plugins.h"

#include <cuda_runtime_api.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
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
static void dump(const char* name, const std::vector<unsigned char>& b) {
    std::printf("blob %s ", name);
    for (unsigned char c : b) std::printf("%02x", c);
    std::printf("\n");
}
static const YoloCore& core_of(IPluginV2* p) { return dynamic_cast<YoloLayerPluginDynamic*>(p)->core(); }

// createPlugin of one field -> the plugin, round trip through both adapters' deserializePlugin; returns the blob
template <int Driver>
static std::vector<unsigned char> round_trip(const PluginField& f, int det_floats, int levels) {
    YoloAnchorFreeCreatorT<Driver, true> cr;
    YoloAnchorFreeCreatorT<Driver, false> cr_io;
    cr.setPluginNamespace("ns1");
    PluginFieldCollection fc{1, &f};
    IPluginV2* p = cr.createPlugin("yololayer", &fc);
    CHECK(p != nullptr && std::strcmp(p->getPluginNamespace(), "ns1") == 0 && std::strcmp(p->getPluginType(), "YoloLayer_TRT") == 0);
    const trtx_yolo_params& q = core_of(p).p;
    const int* v = static_cast<const int*>(f.data);
    CHECK(q.variant == TRTX_YOLO_V8 && q.num_classes == v[0] && q.net_w == v[1] && q.net_h == v[2] && q.max_out == v[3]);
    CHECK(q.det_floats == det_floats && q.num_levels == levels && q.num_kpts == 0 && !q.is_pose && !q.is_obb);
    for (int i = 0; i < levels; ++i) CHECK(q.strides[i] > 0 && q.grid_w[i] == v[1] / q.strides[i] && q.grid_h[i] == v[2] / q.strides[i]);
    CHECK(core_of(p).out_elems() == 1 + v[3] * det_floats);
    const std::vector<unsigned char> b = blob_of(p);
    CHECK(b.size() == (Driver == 9 ? 21u : 24u + 4u * levels));
    int tc;
    std::memcpy(&tc, b.data() + 4, 4);
    CHECK(tc == 256);
    IPluginV2* pio = cr_io.createPlugin("yololayer", &fc);
    CHECK(pio != nullptr && dynamic_cast<YoloLayerPluginIOExt*>(pio) != nullptr && blob_of(pio) == b);
    auto* io = dynamic_cast<IPluginV2IOExt*>(pio);
    CHECK(io->getOutputDimensions(0, nullptr, 0).d[0] == 1 + v[3] * det_floats);
    pio->destroy();
    for (int dyn = 0; dyn < 2; ++dyn) {
        IPluginV2* r = dyn ? cr.deserializePlugin("yololayer", b.data(), b.size()) : cr_io.deserializePlugin("yololayer", b.data(), b.size());
        CHECK(r != nullptr && blob_of(r) == b);
        if (dyn) CHECK(std::memcmp(&core_of(r).p, &q, sizeof(q)) == 0);
        r->destroy();
    }
    // threadCount travels through the blob
    std::vector<unsigned char> b2 = b;
    const int tc2 = 64;
    std::memcpy(b2.data() + 4, &tc2, 4);
    IPluginV2* r = cr.deserializePlugin("yololayer", b2.data(), b2.size());
    CHECK(r != nullptr && blob_of(r) == b2);
    r->destroy();
    // lengths other than the layout's own are refused, never asserted on
    std::vector<unsigned char> big(b.size() + 64, 0);
    std::memcpy(big.data(), b.data(), b.size());
    for (size_t len : {(size_t)0, (size_t)4, (size_t)20, (size_t)23, b.size() - 4, b.size() - 1, b.size() + 1, b.size() + 4, b.size() + 8})
        if (len != b.size()) CHECK(cr.deserializePlugin("yololayer", big.data(), len) == nullptr);
    CHECK(cr.deserializePlugin("yololayer", nullptr, b.size()) == nullptr);
    p->destroy();
    return b;
}

static void check_host(bool print) {
    // the registry holds the creator TRTX_YOLO_ANCHOR_FREE selects, under the reference's name
    IPluginCreator* reg = getPluginRegistry()->getPluginCreator("YoloLayer_TRT", "1");
    CHECK(reg != nullptr && dynamic_cast<YoloV9PluginCreator*>(reg) != nullptr);

    // yolov9: "netinfo" = {nc, w, h, maxOut, is_seg}, declared kFLOAT32 by the builder (block.cpp:405-410)
    const int ni[2][5] = {{80, 640, 640, 2000, 0}, {80, 640, 640, 2000, 1}};
    const char* v9_names[2] = {"yolov9", "yolov9-seg"};
    for (int s = 0; s < 2; ++s) {
        PluginField f("netinfo", ni[s], PluginFieldType::kFLOAT32, 5);
        const std::vector<unsigned char> b = round_trip<9>(f, 38, 3);
        CHECK(b[20] == s);
        if (print) dump(v9_names[s], b);
        PluginField fi("netinfo", ni[s], PluginFieldType::kINT32, 5);  // the type is not looked at
        PluginFieldCollection fc{1, &fi};
        IPluginV2* p = YoloV9PluginCreator().createPlugin("yololayer", &fc);
        CHECK(p != nullptr && blob_of(p) == b && core_of(p).p.is_seg == s);
        p->destroy();
        std::vector<unsigned char> bad = b;  // an is_seg byte that is no bool
        bad[20] = 2;
        CHECK(YoloV9PluginCreator().deserializePlugin("yololayer", bad.data(), bad.size()) == nullptr);
    }
    // yolov10 / yolov13: "combinedInfo" = {nc, w, h, maxOut, strides...}
    const int ci[7] = {80, 640, 640, 1000, 8, 16, 32};
    PluginField f10("combinedInfo", ci, PluginFieldType::kINT32, 7);
    const std::vector<unsigned char> b10 = round_trip<10>(f10, 6, 3);
    if (print) dump("yolov10", b10);
    const int ci4[8] = {2, 1280, 1280, 300, 8, 16, 32, 64};  // another class count, size and level count
    PluginField f4("combinedInfo", ci4, PluginFieldType::kINT32, 8);
    round_trip<10>(f4, 6, 4);
    int ci8[12] = {80, 640, 640, 1000, 8, 8, 8, 8, 8, 8, 8, 8};
    PluginField f8("combinedInfo", ci8, PluginFieldType::kINT32, 12);
    round_trip<10>(f8, 6, 8);

    // malformed field collections are refused
    YoloV9PluginCreator c9;
    YoloV10PluginCreator c10;
    PluginFieldCollection empty{0, nullptr};
    CHECK(c9.createPlugin("y", nullptr) == nullptr && c9.createPlugin("y", &empty) == nullptr);
    CHECK(c10.createPlugin("y", nullptr) == nullptr && c10.createPlugin("y", &empty) == nullptr);
    PluginField short9("netinfo", ni[0], PluginFieldType::kFLOAT32, 4), named9("combinedInfo", ni[0], PluginFieldType::kFLOAT32, 5),
        null9("netinfo", nullptr, PluginFieldType::kFLOAT32, 5), anon9(nullptr, ni[0], PluginFieldType::kFLOAT32, 5);
    for (const PluginField* f : {&short9, &named9, &null9, &anon9}) {
        PluginFieldCollection fc{1, f};
        CHECK(c9.createPlugin("y", &fc) == nullptr);
    }
    PluginField two[2] = {PluginField("netinfo", ni[0], PluginFieldType::kFLOAT32, 5), PluginField("kernels", ni[0], PluginFieldType::kFLOAT32, 1)};
    PluginFieldCollection fc2{2, two};
    CHECK(c9.createPlugin("y", &fc2) == nullptr);
    int ci9[13] = {80, 640, 640, 1000, 8, 8, 8, 8, 8, 8, 8, 8, 8};
    const int zero_stride[7] = {80, 640, 640, 1000, 8, 0, 32}, neg_stride[7] = {80, 640, 640, 1000, 8, 16, -32};
    PluginField no_strides("combinedInfo", ci, PluginFieldType::kINT32, 4), nine("combinedInfo", ci9, PluginFieldType::kINT32, 13),
        zero("combinedInfo", zero_stride, PluginFieldType::kINT32, 7), neg("combinedInfo", neg_stride, PluginFieldType::kINT32, 7),
        named10("netinfo", ci, PluginFieldType::kINT32, 7);
    for (const PluginField* f : {&no_strides, &nine, &zero, &neg, &named10}) {
        PluginFieldCollection fc{1, f};
        CHECK(c10.createPlugin("y", &fc) == nullptr);
    }
    // blobs: a v10 blob whose level count disagrees with its length, zero / negative strides, the other driver's blob
    std::vector<unsigned char> b = b10;
    const int n_bad[4] = {0, -1, 4, 9};
    for (int n : n_bad) {
        std::vector<unsigned char> x = b;
        std::memcpy(x.data() + 20, &n, 4);
        CHECK(c10.deserializePlugin("y", x.data(), x.size()) == nullptr);
    }
    for (int v : {0, -8}) {
        std::vector<unsigned char> x = b;
        std::memcpy(x.data() + 28, &v, 4);
        CHECK(c10.deserializePlugin("y", x.data(), x.size()) == nullptr);
    }
    {
        PluginField f("netinfo", ni[0], PluginFieldType::kFLOAT32, 5);
        PluginFieldCollection fc{1, &f};
        IPluginV2* p9 = c9.createPlugin("y", &fc);
        const std::vector<unsigned char> b9 = blob_of(p9);
        p9->destroy();
        CHECK(c10.deserializePlugin("y", b9.data(), b9.size()) == nullptr);
        CHECK(c9.deserializePlugin("y", b10.data(), b10.size()) == nullptr);
        // the generic creator is unchanged: it refuses both fields (yolov9 has no "kernels", a 7-int combinedInfo is no
        // yolov8 one) and both blobs (21 and 36 bytes are none of its layouts)
        YoloPluginCreator gen;
        CHECK(gen.createPlugin("y", &fc) == nullptr);
        PluginFieldCollection fc10{1, &f10};
        CHECK(gen.createPlugin("y", &fc10) == nullptr);
        CHECK(gen.deserializePlugin("y", b9.data(), b9.size()) == nullptr);
        CHECK(gen.deserializePlugin("y", b10.data(), b10.size()) == nullptr);
    }
}

// enqueue through both adapters == trtx_yolo_decode_enqueue on the plugin's own parameters
template <int Driver>
static void check_gpu(const PluginField& f, const char* name) {
    const int batch = 3;
    YoloAnchorFreeCreatorT<Driver, true> cr;
    YoloAnchorFreeCreatorT<Driver, false> cr_io;
    PluginFieldCollection fc{1, &f};
    auto* dyn = static_cast<YoloLayerPluginDynamic*>(cr.createPlugin("yololayer", &fc));
    auto* io = static_cast<YoloLayerPluginIOExt*>(cr_io.createPlugin("yololayer", &fc));
    const trtx_yolo_params q = dyn->core().p;
    const int C = 4 + q.num_classes + (q.is_seg ? 32 : 0);
    std::mt19937 rng(23);
    std::normal_distribution<float> nd(-4.0f, 2.0f);
    std::vector<void*> in(q.num_levels);
    std::vector<PluginTensorDesc> desc(q.num_levels);
    for (int l = 0; l < q.num_levels; ++l) {
        std::vector<float> h((size_t)batch * C * q.grid_h[l] * q.grid_w[l]);
        for (auto& v : h) v = nd(rng);
        CHECK(cudaMalloc(&in[l], h.size() * 4) == cudaSuccess);
        CHECK(cudaMemcpy(in[l], h.data(), h.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess);
        desc[l].dims.nbDims = 3;
        desc[l].dims.d[0] = batch;
        desc[l].dims.d[1] = C;
        desc[l].dims.d[2] = q.grid_h[l] * q.grid_w[l];
        desc[l].type = DataType::kFLOAT;
        desc[l].format = TensorFormat::kLINEAR;
    }
    const size_t out_n = (size_t)batch * (1 + q.max_out * q.det_floats);
    const size_t ws_n = trtx_yolo_workspace_size(&q, batch);
    CHECK(ws_n > 0 && dyn->getWorkspaceSize(desc.data(), q.num_levels, nullptr, 1) >= ws_n && io->getWorkspaceSize(batch) >= ws_n);
    void *ws, *m[3];
    CHECK(cudaMalloc(&ws, ws_n) == cudaSuccess);
    for (auto& p : m) CHECK(cudaMalloc(&p, out_n * 4) == cudaSuccess && cudaMemset(p, 0, out_n * 4) == cudaSuccess);
    CHECK(trtx_yolo_decode_enqueue(&q, batch, in.data(), static_cast<float*>(m[0]), ws, ws_n, nullptr) == 0);
    void* outs_dyn[1] = {m[1]};
    CHECK(dyn->enqueue(desc.data(), nullptr, in.data(), outs_dyn, ws, nullptr) == 0);
    void* outs_io[1] = {m[2]};
    CHECK(io->enqueue(batch, in.data(), outs_io, ws, nullptr) == 0);
    CHECK(cudaDeviceSynchronize() == cudaSuccess);
    std::vector<float> a(out_n), b(out_n), c(out_n);
    cudaMemcpy(a.data(), m[0], out_n * 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(b.data(), m[1], out_n * 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(c.data(), m[2], out_n * 4, cudaMemcpyDeviceToHost);
    CHECK(a[0] > 0 && std::memcmp(a.data(), b.data(), out_n * 4) == 0 && std::memcmp(a.data(), c.data(), out_n * 4) == 0);
    std::printf("%s gpu rows %d\n", name, (int)a[0]);
    for (void* p : in) cudaFree(p);
    for (void* p : m) cudaFree(p);
    cudaFree(ws);
    dyn->destroy();
    io->destroy();
}

int main(int argc, char** argv) {
    const bool print = argc > 1 && std::strcmp(argv[1], "--dump") == 0;
    const bool gpu = argc > 1 && std::strcmp(argv[1], "--gpu") == 0;
    check_host(print);
    std::printf("anchor-free adapter check ok\n");
    if (gpu) {
        const int ni[5] = {80, 640, 640, 2000, 1};
        check_gpu<9>(PluginField("netinfo", ni, PluginFieldType::kFLOAT32, 5), "yolov9-seg");
        const int ci[7] = {80, 640, 640, 1000, 8, 16, 32};
        check_gpu<10>(PluginField("combinedInfo", ci, PluginFieldType::kINT32, 7), "yolov10");
        std::printf("gpu enqueue ok\n");
    }
    return 0;
}
