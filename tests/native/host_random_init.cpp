// lsd_host.h's DepthMap::initializeRandomly in a process of its own, as main_on_images.cpp:242 reaches it through
// SlamSystem::randomInit: srand(seed) (or initstate(seed, buf, size) for another state type), k calls of rand(), then the adapter's
// initializeRandomly on one image.  Used by tests/test_gpu_random_init.py.
//
//   host_random_init IMAGE.bin OUT.bin SEED K SIZE        SIZE = 0: srand(SEED); otherwise initstate(SEED, buf, SIZE)
//
// IMAGE.bin: int32 w, h; float K[9]; uint8 image [w*h].  OUT.bin: the next 1000 rand() values (int32), then the depth map
// (w*h lsdgpu_hyp records).
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../lsd_slam_b200/host/lsd_host.h"
using namespace lsd_slam;

int main(int argc, char** argv)
{
    if (argc != 6) { std::fprintf(stderr, "usage: %s IMAGE.bin OUT.bin SEED K SIZE\n", argv[0]); return 2; }
    const unsigned seed = (unsigned)std::strtoul(argv[3], nullptr, 10);
    const long k = std::strtol(argv[4], nullptr, 10);
    const int size = std::atoi(argv[5]);
    FILE* f = std::fopen(argv[1], "rb");
    if (!f) { std::perror(argv[1]); return 2; }
    int wh[2];
    Matrix3f K;
    bool ok = std::fread(wh, 4, 2, f) == 2 && std::fread(K.m, 4, 9, f) == 9;
    const int w = wh[0], h = wh[1];
    std::vector<unsigned char> image(ok ? (size_t)w * h : 0);
    ok = ok && std::fread(image.data(), 1, image.size(), f) == image.size();
    std::fclose(f);
    if (!ok) { std::fprintf(stderr, "%s: short file\n", argv[1]); return 2; }

    static int32_t buf[64];
    if (size) initstate(seed, (char*)buf, size);
    else srand(seed);
    for (long i = 0; i < k; i++) (void)rand();

    std::vector<int32_t> next(1000);
    std::vector<lsdgpu_hyp> map;
    try {
        DeviceContext dev(0, w, h, K, 4);
        Frame frame(dev, 0, w, h, K, 0.0, image.data());
        DepthMap dm(dev, w, h, K);
        dm.initializeRandomly(&frame);
        for (int32_t& v : next) v = rand();
        dm.download(map);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "%s\n", e.what());
        return 1;
    }
    FILE* o = std::fopen(argv[2], "wb");
    if (!o) { std::perror(argv[2]); return 2; }
    std::fwrite(next.data(), 4, next.size(), o);
    std::fwrite(map.data(), sizeof(lsdgpu_hyp), map.size(), o);
    std::fclose(o);
    return 0;
}
