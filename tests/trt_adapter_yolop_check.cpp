// trt_adapter_yolop_check.cpp -- the YoloLayer_TRT creator of include/trtx_plugins.h driven with the yolov7 and YOLOP field
// collections and plan blobs.  Built with -fsanitize=address against tests/mock_trt/NvInfer.h, every field in a heap buffer
// of exactly its declared length (YOLOP's netdata: the 4 ints its builder stores), so that a read past a field fails.
// --dump prints the serialized blobs for tests/test_yolop_cpu.py to compare with the Python mirror.
#include "trtx_plugins.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
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

// fields whose data live in heap buffers of exactly `ints` ints
struct Fields {
    std::vector<std::unique_ptr<int[]>> bufs;
    std::vector<std::string> names;
    std::vector<PluginField> f;
    void add(const char* name, std::vector<int> v, int declared) {
        bufs.emplace_back(new int[v.size()]);
        std::memcpy(bufs.back().get(), v.data(), v.size() * sizeof(int));
        names.emplace_back(name);
        f.emplace_back(nullptr, bufs.back().get(), PluginFieldType::kFLOAT32, declared);
    }
    void add(const char* name, std::vector<int> v) { add(name, v, (int)v.size()); }
    PluginFieldCollection fc() {
        for (size_t i = 0; i < f.size(); ++i) f[i].name = names[i].c_str();
        return PluginFieldCollection{(int32_t)f.size(), f.data()};
    }
};

// YOLOP's anchors (yolop/yolop.py: 3,9,5,11,4,20 | 7,18,6,39,12,31 | 19,50,38,81,68,157) and grids for 640 x 384
static const int kYolopAnchors[3][6] = {{3, 9, 5, 11, 4, 20}, {7, 18, 6, 39, 12, 31}, {19, 50, 38, 81, 68, 157}};

// the collection of yolop/common.hpp:318-356: netdata declared 3, carrying 4; yolodataK = stride 8 * 2^(K-1)
static Fields yolop_fields(int order_shift = 0) {
    Fields f;
    std::vector<std::pair<std::string, std::vector<int>>> kernels;
    const int scale[3] = {8, 16, 32};
    for (int k = 0; k < 3; ++k) {
        std::vector<int> d = {640 / scale[k], 384 / scale[k]};
        for (int j = 0; j < 6; ++j) d.push_back(kYolopAnchors[k][j]);
        kernels.emplace_back("yolodata" + std::to_string(k + 1), d);
    }
    if (order_shift == 0) f.add("netdata", {1, 640, 384, 1000}, 3);
    for (int k = 0; k < 3; ++k) {
        const auto& kv = kernels[(k + order_shift) % 3];
        f.add(kv.first.c_str(), kv.second);
    }
    if (order_shift != 0) f.add("netdata", {1, 640, 384, 1000}, 3);
    return f;
}

template <bool Dynamic>
static std::vector<char> blob_of(IPluginV2* p) {
    CHECK(p != nullptr);
    std::vector<char> b(p->getSerializationSize());
    p->serialize(b.data());
    return b;
}

static void dump(const char* name, const std::vector<char>& b) {
    std::printf("blob %s ", name);
    for (char c : b) std::printf("%02x", (unsigned char)c);
    std::printf("\n");
}

template <bool Dynamic>
static IPluginV2* create(Fields& f) {
    YoloPluginCreatorT<Dynamic> c;
    PluginFieldCollection fc = f.fc();
    return c.createPlugin("yololayer", &fc);
}

template <bool Dynamic>
static void round_trip(const std::vector<char>& b) {
    YoloPluginCreatorT<Dynamic> c;
    IPluginV2* q = c.deserializePlugin("yololayer", b.data(), b.size());
    CHECK(q != nullptr);
    CHECK(blob_of<Dynamic>(q) == b);
    q->destroy();
}

int main(int argc, char** argv) {
    const bool dump_blobs = argc > 1 && std::strcmp(argv[1], "--dump") == 0;

    // ---- YOLOP's collection (IOExt: YOLOP's builder is implicit-batch) and the same fields in another order ----
    Fields yf = yolop_fields();
    IPluginV2* yolop = create<false>(yf);
    CHECK(yolop != nullptr);
    const std::vector<char> yb = blob_of<false>(yolop);
    CHECK(yb.size() == 24 + 32 * 3);
    CHECK(static_cast<YoloLayerPluginIOExt*>(yolop)->getOutputDimensions(0, nullptr, 0).d[0] == 1 + 1000 * 6);
    Fields yf2 = yolop_fields(1);
    IPluginV2* yolop2 = create<false>(yf2);
    CHECK(yolop2 != nullptr && blob_of<false>(yolop2) == yb);
    // the dynamic form comes from the same core
    Fields yf3 = yolop_fields();
    IPluginV2* yolop_dyn = create<true>(yf3);
    CHECK(yolop_dyn != nullptr && blob_of<true>(yolop_dyn) == yb);

    // ---- yolov7's collection: netinfo of 4 ints + kernels (yolov7/src/block.cpp:224-241) ----
    float kern[3][8];
    const int scale[3] = {8, 16, 32};
    const float v7_anchors[3][6] = {{12, 16, 19, 36, 40, 28}, {36, 75, 76, 55, 72, 146}, {142, 110, 192, 243, 459, 401}};
    for (int k = 0; k < 3; ++k) {
        const int gw = 640 / scale[k], gh = 640 / scale[k];
        std::memcpy(&kern[k][0], &gw, 4);
        std::memcpy(&kern[k][1], &gh, 4);
        for (int j = 0; j < 6; ++j) kern[k][2 + j] = v7_anchors[k][j];
    }
    auto v7_fields = [&](int netinfo_len) {
        Fields f;
        std::vector<int> ni = {80, 640, 640, 1000, 0};
        ni.resize(netinfo_len);
        f.add("netinfo", ni);
        std::vector<int> kv(24);
        std::memcpy(kv.data(), kern, sizeof(kern));
        f.add("kernels", kv, 3);  // length = number of YoloKernel
        return f;
    };
    Fields v7f = v7_fields(4);
    IPluginV2* v7 = create<true>(v7f);
    CHECK(v7 != nullptr);
    const std::vector<char> v7b = blob_of<true>(v7);
    CHECK(v7b.size() == 24 + 32 * 3);
    // yolov5's netinfo of 5: unchanged
    Fields v5f = v7_fields(5);
    IPluginV2* v5 = create<true>(v5f);
    CHECK(v5 != nullptr);
    const std::vector<char> v5b = blob_of<true>(v5);
    CHECK(v5b.size() == 25 + 32 * 3);

    // ---- v8 combinedInfo: unchanged ----
    Fields v8f;
    v8f.add("combinedInfo", {80, 17, 0, 640, 640, 1000, 0, 0, 0, 8, 16, 32});
    IPluginV2* v8 = create<true>(v8f);
    CHECK(v8 != nullptr);
    const std::vector<char> v8b = blob_of<true>(v8);
    CHECK(v8b.size() == 35 + 4 * 3);

    // ---- every blob deserializes to the same plugin, in both forms; the three layouts are 3, 1 and 0 mod 4 ----
    CHECK(v8b.size() % 4 == 3 && v5b.size() % 4 == 1 && yb.size() % 4 == 0);
    for (const auto* b : {&yb, &v7b, &v5b, &v8b}) {
        round_trip<true>(*b);
        round_trip<false>(*b);
    }
    // blobs of lengths no layout has are refused (a length another layout has is that layout's blob: a layout is told
    // apart by its length alone)
    {
        YoloPluginCreator c;
        for (const auto* b : {&yb, &v5b, &v8b})
            for (long extra : {-2L, -1L, 1L, 2L}) {
                const size_t n = b->size() + extra;
                if (n % 4 == 0 ? (n - 24) % 32 == 0 : n % 4 == 1 ? (n - 25) % 32 == 0 : n % 4 == 3) continue;
                std::vector<char> d(*b);
                d.resize(n);
                CHECK(c.deserializePlugin("x", d.data(), d.size()) == nullptr);
            }
        std::vector<char> d(yb);
        d.pop_back();  // 119 bytes: the v8 length class, but not a v8 header
        CHECK(c.deserializePlugin("x", d.data(), d.size()) == nullptr);
    }

    // ---- malformed collections are refused (and, under ASan, never read past a field) ----
    {
        Fields f = yolop_fields();
        f.f.pop_back();  // yolodata3 missing
        f.names.pop_back();
        CHECK(create<false>(f) == nullptr);
    }
    {
        Fields f;
        f.add("netdata", {1, 640}, 2);  // too short
        for (int k = 0; k < 3; ++k) {
            std::vector<int> d = {80 >> k, 48 >> k};
            for (int j = 0; j < 6; ++j) d.push_back(kYolopAnchors[k][j]);
            f.add(("yolodata" + std::to_string(k + 1)).c_str(), d);
        }
        CHECK(create<false>(f) == nullptr);
    }
    {
        Fields f;
        f.add("netdata", {1, 640, 384, 1000}, 3);
        for (int k = 0; k < 3; ++k) {
            std::vector<int> d = {80 >> k, 48 >> k};
            for (int j = 0; j < (k == 1 ? 5 : 6); ++j) d.push_back(kYolopAnchors[k][j]);  // yolodata2 of 7 ints
            f.add(("yolodata" + std::to_string(k + 1)).c_str(), d);
        }
        CHECK(create<false>(f) == nullptr);
    }
    {
        Fields f;
        f.add("netdata", {1, 640, 384, 1000}, 3);
        for (int k = 0; k < 3; ++k) {
            std::vector<int> d = {80 >> k, 48 >> k};
            for (int j = 0; j < 6; ++j) d.push_back(kYolopAnchors[k][j]);
            f.add(k == 2 ? "yolodata1" : ("yolodata" + std::to_string(k + 1)).c_str(), d);  // yolodata1 twice
        }
        CHECK(create<false>(f) == nullptr);
    }
    {
        Fields f;
        f.add("netinfo", {80, 640, 640}, 3);  // too short
        std::vector<int> kv(24);
        std::memcpy(kv.data(), kern, sizeof(kern));
        f.add("kernels", kv, 3);
        CHECK(create<true>(f) == nullptr);
    }
    {
        Fields f;
        f.add("combinedInfo", {80, 17, 0, 640, 640, 1000, 0, 0, 0});  // no stride
        CHECK(create<true>(f) == nullptr);
    }

    if (dump_blobs) {
        dump("yolop", yb);
        dump("yolov7", v7b);
        dump("yolov5", v5b);
        dump("yolov8", v8b);
    }
    for (IPluginV2* p : {yolop, yolop2, yolop_dyn, v7, v5, v8}) p->destroy();
    std::printf("trt adapter yolop check ok\n");
    return 0;
}
