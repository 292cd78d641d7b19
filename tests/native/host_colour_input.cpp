// lsd_host.h fed colour camera images: getUndistorterForFile (util/Undistorter.cpp:38-88), install, then the conversion of
// LiveSLAMWrapper::newImageCallback (LiveSLAMWrapper.cpp:116-121) as one DeviceContext::setInputFormat call, then
// Undistorter::undistort and Frame(.., raw, /*distorted=*/true) on the raw colour image.  Used by tests/test_gpu_colour_input_host.py.
//
//   host_colour_input CALIB_FILE CHANNELS FORMAT RAW.bin OUT.bin
//     CHANNELS  the camera image's channel count, as cv::Mat::channels() would report it (1, 2, 3 or 4)
//     FORMAT    the LSDGPU_PIX_* number of a multi-channel image (a 1-channel image is MONO8)
//     RAW.bin   in_height * in_width * CHANNELS bytes
//   OUT.bin: undistort()'s w*h bytes, then the frame's image levels 0..4 (floats) and maxGradients (floats), native byte order
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

#include "../../lsd_slam_b200/host/lsd_host.h"
using namespace lsd_slam;

int main(int argc, char** argv)
{
    if (argc < 6) {
        std::fprintf(stderr, "usage: host_colour_input CALIB_FILE CHANNELS FORMAT RAW.bin OUT.bin\n");
        return 2;
    }
    const int channels = std::atoi(argv[2]), format = std::atoi(argv[3]);
    try {
        std::unique_ptr<Undistorter> u(getUndistorterForFile(argv[1]));
        if (!u) { std::fprintf(stderr, "invalid calibration\n"); return 2; }
        const int w = u->getOutputWidth(), h = u->getOutputHeight();
        std::vector<unsigned char> raw((size_t)u->getInputWidth() * u->getInputHeight() * channels);
        FILE* f = std::fopen(argv[4], "rb");
        if (!f || std::fread(raw.data(), 1, raw.size(), f) != raw.size()) { std::fprintf(stderr, "cannot read %s\n", argv[4]); return 2; }
        std::fclose(f);

        DeviceContext dev(0, w, h, u->getK(), 4);
        u->install(dev);
        dev.setInputFormat(channels == 1 ? LSDGPU_PIX_MONO8 : format);      // newImageCallback's cvtColor, LiveSLAMWrapper.cpp:116-121
        std::vector<unsigned char> undist((size_t)w * h);
        u->undistort(dev, raw.data(), undist.data());
        Frame frame(dev, 1, w, h, u->getK(), 0.0, raw.data(), /*distorted=*/true);

        FILE* o = std::fopen(argv[5], "wb");
        if (!o) return 2;
        std::fwrite(undist.data(), 1, undist.size(), o);
        for (int lvl = 0; lvl < LSDGPU_LEVELS; lvl++) {
            std::vector<float> img((size_t)(w >> lvl) * (h >> lvl));
            dev.check(lsdgpu_frame_download(dev.raw(), 1, LSDGPU_BUF_IMAGE, lvl, img.data()), "download");
            std::fwrite(img.data(), 4, img.size(), o);
        }
        std::vector<float> mg((size_t)w * h);
        dev.check(lsdgpu_frame_download(dev.raw(), 1, LSDGPU_BUF_MAXGRAD, 0, mg.data()), "download");
        std::fwrite(mg.data(), 4, mg.size(), o);
        std::fclose(o);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "host_colour_input: %s\n", e.what());
        return 1;
    }
    return 0;
}
