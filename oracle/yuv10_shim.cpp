// TEST INFRASTRUCTURE - libyuv's portable C rows for the 10-bit path and the BT.2020 / full-range BT.601 matrices, as plain C symbols
// (see yuv10.mk): I210ToAR30Row_C (YuvPixel16 + StoreAR30) and the 8-bit I422ToARGBRow_C (YuvPixel), each with one of four tables:
// 0 kYuvI601Constants, 1 kYuvH709Constants, 2 kYuv2020Constants, 3 kYuvJPEGConstants. Both return 0, or -1 for a bad argument.
#include "libyuv/row.h"

using namespace libyuv;

static const struct YuvConstants* yuv10_table(int sel) {
    switch (sel) {
    case 0: return &kYuvI601Constants;
    case 1: return &kYuvH709Constants;
    case 2: return &kYuv2020Constants;
    case 3: return &kYuvJPEGConstants;
    }
    return nullptr;
}

extern "C" {
int yuv10_i210_ar30_row(const uint16_t* y, const uint16_t* u, const uint16_t* v, uint8_t* dst, int width, int sel) {
    const struct YuvConstants* k = yuv10_table(sel);
    if (!k || !y || !u || !v || !dst || width <= 0) return -1;
    I210ToAR30Row_C(y, u, v, dst, k, width);
    return 0;
}
int yuv10_i422_argb_row(const uint8_t* y, const uint8_t* u, const uint8_t* v, uint8_t* dst, int width, int sel) {
    const struct YuvConstants* k = yuv10_table(sel);
    if (!k || !y || !u || !v || !dst || width <= 0) return -1;
    I422ToARGBRow_C(y, u, v, dst, k, width);
    return 0;
}
}
