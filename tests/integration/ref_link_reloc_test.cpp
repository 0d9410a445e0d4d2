// tests/integration/ref_link_reloc_test.cpp — TEST INFRASTRUCTURE.
// The relocalisation overload ORBmatcher::SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist) inside the linked reference
// build: oracle/ref_link_reloc_build.sh links this file and tests/ref_reloc.cpp (the reference's own Frame / KeyFrame / MapPoint objects
// built from plain arrays) with the objects of oracle/ref_link_build.sh, whose ORBmatcher.cc symbols are weak, so the call runs the
// adapter of structure-slam-pointline_b200/host/matcher_b200.cc and the GPU.  tests/test_integration_reloc_gpu.py writes the scene,
// runs this program and holds its output against tests/reloc_model.py and the reference's own matcher.
//
// usage: ref_link_reloc_test scene.bin out.bin
//   scene.bin: int32 n1, nel, n2, nlevels, ORBdist, checkOri; float32 th, scaleFactor, cam8[8], Tcw[12]; then kp1[n1] (cv::KeyPoint),
//              kfmp[n1] i32, Xw[nel][3], mindist[nel], maxdist[nel] f32, eldesc[nel][32], bad[nel], found[nel], held[n2] u8,
//              kp2[n2] (cv::KeyPoint), d2[n2][32] u8
//   out.bin:   int32 nmatches, assign2[n2] (element index, -1 none, -3 the MapPoint the feature held)
#include <cstdint>
#include <cstdio>
#include <fstream>
#include <vector>

extern "C" int ref_search_by_projection_kf(int n1, const void* kp1, const int32_t* kfmp, int nel, const float* Xw, const float* mindist,
                                           const float* maxdist, const uint8_t* eldesc, const uint8_t* bad, const uint8_t* found,
                                           int n2, const void* kp2, const uint8_t* d2, const uint8_t* held2, const float* Tcw,
                                           const float* cam8, int nlevels, float scaleFactor, float th, int ORBdist, int checkOri,
                                           int32_t* assign2, double* seconds);

template <class T> static std::vector<T> take(std::ifstream& f, size_t n) {
    std::vector<T> v(n + 1);
    f.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * sizeof(T)));
    return v;
}

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: ref_link_reloc_test scene.bin out.bin\n"); return 2; }
    std::ifstream f(argv[1], std::ios::binary);
    if (!f) { fprintf(stderr, "cannot read %s\n", argv[1]); return 2; }
    const std::vector<int32_t> h = take<int32_t>(f, 6);
    const int n1 = h[0], nel = h[1], n2 = h[2];
    const std::vector<float> p = take<float>(f, 22);
    const std::vector<uint8_t> kp1 = take<uint8_t>(f, (size_t)n1 * 28);
    const std::vector<int32_t> kfmp = take<int32_t>(f, n1);
    const std::vector<float> Xw = take<float>(f, (size_t)nel * 3), mind = take<float>(f, nel), maxd = take<float>(f, nel);
    const std::vector<uint8_t> eldesc = take<uint8_t>(f, (size_t)nel * 32), bad = take<uint8_t>(f, nel), found = take<uint8_t>(f, nel),
                               held = take<uint8_t>(f, n2), kp2 = take<uint8_t>(f, (size_t)n2 * 28), d2 = take<uint8_t>(f, (size_t)n2 * 32);
    if (!f) { fprintf(stderr, "short scene file\n"); return 2; }
    std::vector<int32_t> out(n2 + 1);
    out[0] = ref_search_by_projection_kf(n1, kp1.data(), kfmp.data(), nel, Xw.data(), mind.data(), maxd.data(), eldesc.data(), bad.data(),
                                         found.data(), n2, kp2.data(), d2.data(), held.data(), &p[10], &p[2], h[3], p[1], p[0], h[4], h[5],
                                         out.data() + 1, nullptr);
    std::ofstream o(argv[2], std::ios::binary);
    o.write(reinterpret_cast<const char*>(out.data()), (std::streamsize)(out.size() * sizeof(int32_t)));
    printf("ref_link_reloc_test ok: %d matches\n", out[0]);
    return 0;
}
