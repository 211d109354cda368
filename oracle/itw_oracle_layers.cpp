/*
 * itw_oracle_layers.cpp -- CPU ORACLE for mip levels taken from document layers (itw_dds_encode_layers).  TEST INFRASTRUCTURE,
 * NOT PRODUCT.
 *
 * Restates IntelPlugin.cpp's CopyLayersIntoMipMaps for one level, with the plug-in's scalar conversions as
 * oracle/itw_oracle_frontend.cpp already restates them: that file is included here, whole and unchanged, so that both oracles
 * share one statement of FloatToByte / ConvertTo8Bit / ConvertTo16Bit and of the half conversion.  Built into
 * oracle/libitw_oracle_layers.so by oracle/build_oracle_layers.py; only tests/ may load it.
 *
 * PINNING.  tests/test_mips_from_layers.py compares oracle_copy_layer byte for byte with the reference's OWN bodies of
 * CopyLayersIntoMipMaps, CopyFromLayerChannelIntoImage and FillLayerDataToWhite (oracle/_ref/libitw_ref_layers.so, cut by
 * oracle/build_ref_layers.py), and with digests of those bodies committed under tests/golden.
 */
#include "itw_oracle_frontend.cpp"

// ---- mip levels from document layers ----------------------------------------------------------------------------------
// IntelPlugin.cpp:1749-1850 CopyLayersIntoMipMaps for ONE level, with CopyFromLayerChannelIntoImage (:1694-1741) and
// FillLayerDataToWhite (:1664-1689) per texel, then FlipXYChannelNormalMap (:1504-1546) when `flip` (ITW_FRONT_FLIP_*) is set --
// the save path flips level 0 after layer 0 has overwritten it.  `level` = lw x lh tightly packed RGBA8 / RGBA16F texels,
// overwritten in place; `channels` / `alpha` = planes of the document (doc_w elements per row, `depth` bits each) as
// ReadLayerData delivers them.
namespace {
template <class T>
void copy_layer_plane(bool hdr, void* level, int lw, int lh, int doc_w, const T* plane, int c)
{
    for (int y = 0; y < lh; y++)
        for (int x = 0; x < lw; x++) {
            const T v = plane[(size_t)doc_w * y + x];
            const size_t i = ((size_t)lw * y + x) * 4 + c;
            if (hdr) static_cast<uint16_t*>(level)[i] = to16(v);
            else static_cast<uint8_t*>(level)[i] = to8(v);
        }
}
template <>
void copy_layer_plane<float>(bool hdr, void* level, int lw, int lh, int doc_w, const float* plane, int c)
{
    for (int y = 0; y < lh; y++)
        for (int x = 0; x < lw; x++) {
            const float v = plane[(size_t)doc_w * y + x];
            const size_t i = ((size_t)lw * y + x) * 4 + c;
            if (hdr) static_cast<uint16_t*>(level)[i] = to16(v);
            else static_cast<uint8_t*>(level)[i] = to8(v, true);          // ConvertTo8Bit(double, gammaCorrect = true)
        }
}
template <class T>
void copy_layer(bool hdr, void* level, int lw, int lh, int doc_w, const void* const* channels, int channel_count, const void* alpha,
                T white)
{
    for (int c = 0; c < channel_count; c++) copy_layer_plane(hdr, level, lw, lh, doc_w, static_cast<const T*>(channels[c]), c);
    std::vector<T> fill;
    const T* a = static_cast<const T*>(alpha);
    if (!a) {
        fill.assign((size_t)doc_w * lh, white);
        a = fill.data();
    }
    copy_layer_plane(hdr, level, lw, lh, doc_w, a, 3);
}
}  // namespace

extern "C" int oracle_copy_layer(int hdr, void* level, int lw, int lh, int depth, int doc_w, const void* const* channels, int channel_count,
                                 const void* alpha, int has_alpha, unsigned flip)
{
    if (channel_count < 1 || channel_count > 3 || lw > doc_w) return -1;
    const void* a = has_alpha ? alpha : nullptr;
    if (depth == 8) copy_layer<uint8_t>(hdr != 0, level, lw, lh, doc_w, channels, channel_count, a, (uint8_t)255);
    else if (depth == 16) copy_layer<uint16_t>(hdr != 0, level, lw, lh, doc_w, channels, channel_count, a, to16((uint8_t)255));
    else if (depth == 32) copy_layer<float>(hdr != 0, level, lw, lh, doc_w, channels, channel_count, a, 1.0f);
    else return -1;
    for (size_t i = 0; i < (size_t)lw * lh; i++) {
        if (hdr) {
            uint16_t* p = static_cast<uint16_t*>(level) + 4 * i;
            if (flip & ITW_FRONT_FLIP_X) p[0] = half_from_float(1.0f - float_from_half(p[0]));
            if (flip & ITW_FRONT_FLIP_Y) p[1] = half_from_float(1.0f - float_from_half(p[1]));
        } else {
            uint8_t* p = static_cast<uint8_t*>(level) + 4 * i;
            if (flip & ITW_FRONT_FLIP_X) p[0] = (uint8_t)(255 - p[0]);
            if (flip & ITW_FRONT_FLIP_Y) p[1] = (uint8_t)(255 - p[1]);
        }
    }
    return 0;
}
