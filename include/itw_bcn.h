/*
 * itw_bcn.h -- C-ABI of the H100 (sm_90a) BCn block encoder (libitw_bcn.so).
 *
 * Drop-in boundary: every struct and entry point in the first section has the exact layout,
 * name, argument meaning and calling convention of the reference's
 *     3rdParty/Intel/Source/ispc_texcomp.h:19-50  (structs)
 *     3rdParty/Intel/Source/ispc_texcomp.h:67-87  (GetProfile_*)
 *     3rdParty/Intel/Source/ispc_texcomp.h:104-107 (CompressBlocksBC1/BC3/BC6H/BC7)
 * so a host that links ispc_texcomp today (IntelPlugin.cpp's save path through
 * win32Threads.cpp:289-330) can link this library instead.  The second section is additive.
 *
 * Plain pointers and sizes only; no C++ or torch types cross this boundary.
 */
#ifndef ITW_BCN_H
#define ITW_BCN_H

#include <stdint.h>
#include <stdbool.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------
 * Section 1 -- the reference's own ABI
 * ------------------------------------------------------------------------------------------- */

/* ispc_texcomp.h:19-25.  `stride` is in BYTES.  LDR surfaces are RGBA8 (R in byte 0), HDR
 * surfaces are RGBA16F (half R,G,B at +0,+2,+4; A ignored).  width/height multiples of 4. */
typedef struct rgba_surface {
    uint8_t* ptr;
    int32_t  width;
    int32_t  height;
    int32_t  stride;
} rgba_surface;

/* ispc_texcomp.h:27-41 (64 bytes) */
typedef struct bc7_enc_settings {
    bool mode_selection[4];      /* {modes 0+2, modes 1+3+7, modes 4+5, mode 6} */
    int  refineIterations[8];    /* per BC7 mode */
    bool skip_mode2;
    int  fastSkipTreshold_mode1; /* (sic) number of ranked 2-subset partitions tried */
    int  fastSkipTreshold_mode3;
    int  fastSkipTreshold_mode7;
    int  mode45_channel0;        /* first rotation tried by modes 4/5 */
    int  refineIterations_channel;
    int  channels;               /* 3 = ignore alpha, 4 = RGBA */
} bc7_enc_settings;

/* ispc_texcomp.h:43-50 (16 bytes) */
typedef struct bc6h_enc_settings {
    bool slow_mode;
    bool fast_mode;
    int  refineIterations_1p;
    int  refineIterations_2p;
    int  fastSkipTreshold;
} bc6h_enc_settings;

/* ispc_texcomp.h:67-71 -- RGB profiles (alpha ignored); ispc_texcomp.cpp:20-189 */
void GetProfile_ultrafast(bc7_enc_settings* settings);
void GetProfile_veryfast(bc7_enc_settings* settings);
void GetProfile_fast(bc7_enc_settings* settings);
void GetProfile_basic(bc7_enc_settings* settings);
void GetProfile_slow(bc7_enc_settings* settings);
/* ispc_texcomp.h:74-78 -- RGBA profiles; ispc_texcomp.cpp:191-365 */
void GetProfile_alpha_ultrafast(bc7_enc_settings* settings);
void GetProfile_alpha_veryfast(bc7_enc_settings* settings);
void GetProfile_alpha_fast(bc7_enc_settings* settings);
void GetProfile_alpha_basic(bc7_enc_settings* settings);
void GetProfile_alpha_slow(bc7_enc_settings* settings);
/* ispc_texcomp.h:81-85 -- BC6H profiles; ispc_texcomp.cpp:367-410 */
void GetProfile_bc6h_veryfast(bc6h_enc_settings* settings);
void GetProfile_bc6h_fast(bc6h_enc_settings* settings);
void GetProfile_bc6h_basic(bc6h_enc_settings* settings);
void GetProfile_bc6h_slow(bc6h_enc_settings* settings);
void GetProfile_bc6h_veryslow(bc6h_enc_settings* settings);

/* ispc_texcomp.h:104-107; ispc_texcomp.cpp:417-435 -> kernel.ispc:598/607/3132/2030.
 * dst receives (width/4)*(height/4) blocks, tightly packed in raster block order
 * (8 bytes/block for BC1, 16 for BC3/BC6H/BC7).  `src->ptr` and `dst` may each be host or
 * device memory (detected per call).  The call is synchronous.  With a device operand the work is
 * issued on the legacy default stream, i.e. it is ordered after work already enqueued on blocking
 * streams; producers on NON-blocking streams must be synchronised by the caller (or use
 * itw_encode_device, which is stream-ordered).
 * void return as in the reference: failures are reported through itw_get_last_error(). */
void CompressBlocksBC1(const rgba_surface* src, uint8_t* dst);
void CompressBlocksBC3(const rgba_surface* src, uint8_t* dst);
void CompressBlocksBC6H(const rgba_surface* src, uint8_t* dst, bc6h_enc_settings* settings);
void CompressBlocksBC7(const rgba_surface* src, uint8_t* dst, bc7_enc_settings* settings);

/* ---------------------------------------------------------------------------------------------
 * Section 2 -- additive entry points (not in the reference header)
 * ------------------------------------------------------------------------------------------- */

/* BC4 (R -> 8 B/block) and BC5 (R,G -> 16 B/block) of an RGBA8 surface.  In the reference these
 * formats go through DirectX::Compress (IntelPlugin.cpp:272) to D3DXEncodeBC4U / D3DXEncodeBC5U
 * (DirectXTex/BC4BC5.cpp:403, :481); same surface/dst conventions as above. */
void CompressBlocksBC4(const rgba_surface* src, uint8_t* dst);
void CompressBlocksBC5(const rgba_surface* src, uint8_t* dst);

/* Format selector for the generic entry points below; values are the DXGI_FORMAT enumerants the
 * plug-in switches on (IntelPlugin.cpp:820-847, win32Threads.cpp:192-209). */
enum {
    ITW_FORMAT_BC1 = 71,  /* DXGI_FORMAT_BC1_UNORM  */
    ITW_FORMAT_BC3 = 77,  /* DXGI_FORMAT_BC3_UNORM  */
    ITW_FORMAT_BC4 = 80,  /* DXGI_FORMAT_BC4_UNORM  */
    ITW_FORMAT_BC5 = 83,  /* DXGI_FORMAT_BC5_UNORM  */
    ITW_FORMAT_BC6H = 95, /* DXGI_FORMAT_BC6H_UF16  */
    ITW_FORMAT_BC6H_SF16 = 96, /* DXGI_FORMAT_BC6H_SF16: ENCODED by the same unsigned encoder, as the plug-in does
                                  (IntelPlugin.cpp:840-843); DECODED with the signed rules (DirectXTexCompress.cpp:414) */
    ITW_FORMAT_BC7 = 98   /* DXGI_FORMAT_BC7_UNORM  */
};

/* Bytes per 4x4 block for a format (win32Threads.cpp:192-209); 0 for an unknown format. */
int itw_bytes_per_block(int format);

/* Device-resident encode on an explicit CUDA stream (cudaStream_t passed as void*; NULL = the
 * legacy default stream).  src->ptr and dst MUST be device pointers; nothing is copied and the
 * call returns as soon as the kernel is enqueued.  `settings` is a bc7_enc_settings* for BC7, a
 * bc6h_enc_settings* for BC6H and ignored otherwise; it is read before the call returns.
 * Returns 0 on success, a negative value on error (see itw_get_last_error). */
int itw_encode_device(int format, const rgba_surface* src, uint8_t* dst, const void* settings,
                      void* cuda_stream);

/* Batched encode of `count` independent surfaces (config C5's tile stream).  Host surfaces are pipelined
 * H2D / encode / D2H over internal streams (and dealt round-robin over the devices of itw_set_devices);
 * dst[i] receives surface i's blocks.  Synchronous.  Ordering: device-resident operands are ordered after the work
 * already enqueued on the legacy default stream / blocking streams at the time of the call (as for
 * CompressBlocks*); producers on NON-blocking streams must be synchronised by the caller.  The same rule holds for the
 * device-resident surfaces of itw_dds_encode_file / itw_dds_encode_texture / itw_dds_encode_pixels. */
int itw_encode_batch(int format, const rgba_surface* srcs, uint8_t* const* dsts, int count,
                     const void* settings);

/* Select the CUDA device used by this thread's subsequent calls (default: current device). */
int itw_set_device(int device);

/* Multi-GPU in ONE process (SURVEY.md 8e; the analogue of the reference's thread pool, win32Threads.cpp:98-274, which
 * fans row bands of one surface over its workers, :211-249).  After itw_set_devices(list, n >= 2) every HOST -> HOST
 * call of CompressBlocks* / CompressImage* is cut into one band of whole block rows per device; each device copies
 * in, encodes and copies out its band on its own PCIe link, straight into the caller's dst.  itw_encode_batch deals
 * its tiles round-robin over the devices (config C5's tile stream).  Bands and tiles are independent, so the output is
 * byte-identical to the single-device one; there is no collective.  Device-resident operands stay on their device.
 * n == 1 makes that device the process-wide default; n == 0 restores the single-device behaviour (the calling
 * thread's current device / itw_set_device).  Process-wide; not to be called concurrently with encodes.
 * Returns 0 on success. */
int itw_set_devices(const int* devices, int count);
/* The devices selected by itw_set_devices (written to devices[0..capacity)); returns their number, 0 if none. */
int itw_get_devices(int* devices, int capacity);

/* Deferred mode for hosts that keep the reference's slice loop (IntelPlugin.cpp:851-879: one CompressImageMT per
 * 256 K-texel slice of the image).  Between itw_begin_deferred() and itw_flush(), host -> host encodes issued by the
 * calling thread are only ENQUEUED (copy-in, kernel, copy-out on internal streams, pipelined over three lanes) and
 * return at once; src and dst must stay valid and untouched until itw_flush(), which waits for all of them and returns
 * 0 or the first failure (text in itw_get_last_error).  Two added lines in the host: begin before the loop, flush after. */
int itw_begin_deferred(void);
int itw_flush(void);

/* ---- the reference's coarse seam: 3rdParty/Intel/Source/win32Threads.h:24, :52-80 (win32Threads.cpp:192-330) ----
 * Same names and argument meaning; BYTE is spelled uint8_t and DXGI_FORMAT is passed as int (the enum's underlying
 * type).  CompressImageBC* = GetProfile + CompressBlocks* (win32Threads.cpp:289-330).  CompressImageMT / ST call
 * `cmpFunc` ONCE for the whole surface: the reference's per-thread bands (win32Threads.cpp:217-230) become one GPU
 * launch, or one band per device after itw_set_devices / InitWin32Threads -- same bytes, bands being independent. */
typedef void(CompressionFunc)(const rgba_surface* input, uint8_t* output);
int  GetProcessorCount(void);      /* visible CUDA devices, 1 or more (win32Threads.h:52) */
void InitWin32Threads(void);       /* select every visible GPU (itw_set_devices) -- the pool the reference builds here */
void DestroyThreads(void);         /* back to single-device behaviour */
int  GetBytesPerBlock(int dxgi_format);
bool CompressImageMT(const rgba_surface* input, uint8_t* output, CompressionFunc* cmpFunc, int compformat);
bool CompressImageST(const rgba_surface* input, uint8_t* output, CompressionFunc* cmpFunc, int compformat);
void CompressImageBC1(const rgba_surface* input, uint8_t* output);
void CompressImageBC3(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_ultrafast(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_veryfast(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_fast(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_basic(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_slow(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_alpha_ultrafast(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_alpha_veryfast(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_alpha_fast(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_alpha_basic(const rgba_surface* input, uint8_t* output);
void CompressImageBC7_alpha_slow(const rgba_surface* input, uint8_t* output);
void CompressImageBC6H_veryfast(const rgba_surface* input, uint8_t* output);
void CompressImageBC6H_fast(const rgba_surface* input, uint8_t* output);
void CompressImageBC6H_basic(const rgba_surface* input, uint8_t* output);
void CompressImageBC6H_slow(const rgba_surface* input, uint8_t* output);
void CompressImageBC6H_veryslow(const rgba_surface* input, uint8_t* output);

/* Last error message of the calling thread ("" if none).  The CompressBlocks* entry points keep
 * the reference's void signature, so this is the only error channel for them. */
const char* itw_get_last_error(void);

/* Free the calling thread's device buffers, streams and events now (they are otherwise kept for the next
 * call and freed when the thread exits); the next call re-creates what it needs. */
void itw_release(void);

/* Number of kernel launches issued by this library since load (all threads); bench evidence. */
uint64_t itw_kernel_launch_count(void);

/* Device time in milliseconds of the most recent call issued by this thread (encode, decode, convert),
 * measured with CUDA events on the launching stream around the kernel(s) only (no copies).  For host
 * surfaces BC7 / BC6H run as four pipelined row bands: the span then covers the four kernels including
 * the short waits for the later bands' input copies.  Valid after the call has completed. */
float itw_last_kernel_ms(void);

/* ---------------------------------------------------------------------------------------------
 * Section 3 -- DDS container (SURVEY.md 8f-1): what IntelPlugin.cpp:2171 obtains from
 * DirectX::SaveToDDSMemory (DirectXTex/DirectXTexDDS.cpp:1611-1815) with header rules of
 * _EncodeDDSHeader (:441-675) and the structures of DirectXTex/DDS.h:40-235.  2-D textures and
 * cube maps of block-compressed formats only.
 * ------------------------------------------------------------------------------------------- */
typedef struct itw_dds_desc {
    uint32_t width, height;   /* top level, texels (need not be multiples of 4) */
    uint32_t mip_levels;      /* >= 1 */
    uint32_t array_size;      /* images per mip level: 1, or 6*n for cube maps */
    uint32_t dxgi_format;     /* DXGI_FORMAT value, e.g. 71 BC1_UNORM, 72 BC1_UNORM_SRGB, 77/78 BC3, 80 BC4_UNORM,
                                 83 BC5_UNORM, 95 BC6H_UF16, 96 BC6H_SF16, 98/99 BC7 */
    uint32_t is_cubemap;      /* 0 / 1 */
} itw_dds_desc;

/* 128 (legacy FourCC header: BC1/BC3/BC4U/BC5U, single image or one cube map) or 148 (with the
 * 'DX10' extension: sRGB variants, BC6H, BC7, arrays); 0 if the description is not supported. */
size_t itw_dds_header_bytes(const itw_dds_desc* desc);
/* Bytes of one image (array item `item`, mip `mip`) and its offset from the start of the file;
 * images are stored item-major, mip-minor, each tightly packed (DirectXTexDDS.cpp:1676-1720). */
size_t itw_dds_image_bytes(const itw_dds_desc* desc, uint32_t mip);
size_t itw_dds_image_offset(const itw_dds_desc* desc, uint32_t item, uint32_t mip);
size_t itw_dds_file_bytes(const itw_dds_desc* desc);
/* Write magic + DDS_HEADER (+ DDS_HEADER_DXT10).  Returns the header size, 0 on error. */
size_t itw_dds_write_header(const itw_dds_desc* desc, uint8_t* dst, size_t capacity);
/* Parse a header written by this library or by DirectXTex.  Returns the payload offset, 0 on error. */
size_t itw_dds_read_header(const uint8_t* src, size_t size, itw_dds_desc* desc);
/* The whole save path for one texture: encode array_size*mip_levels surfaces (item-major, mip-minor,
 * each already padded to multiples of 4 as IntelPlugin.cpp:893-928 does) straight into `file`
 * (capacity >= itw_dds_file_bytes) behind the header.  `settings` as for itw_encode_device.
 * Returns the file size, 0 on error. */
size_t itw_dds_encode_file(const itw_dds_desc* desc, const rgba_surface* images, const void* settings,
                           uint8_t* file, size_t capacity);

/* ---------------------------------------------------------------------------------------------
 * Section 4 -- on-GPU pre-pass (SURVEY.md 8f-2): mip chain + pad-to-4.
 * Level l has max(1,w>>l) x max(1,h>>l) texels and is STORED padded to multiples of 4 by edge replication
 * (IntelPlugin.cpp:893-928), rows tightly packed -- ready to be handed to CompressBlocks*.
 * Filters = DirectXTex's own (non-WIC) generators, which are in the reference tree (DirectXTexMipmaps.cpp:715-905,
 * Filters.h:33-112): the BOX filter ((p0+p1)+p2+p3)*0.25 when width and height of level 0 are powers of two, the two-tap
 * LINEAR filter otherwise (GenerateMipMaps' default choice, :2611-2616), every level re-read from the stored previous one.
 *   itw_generate_mips_device       RGBA8 as R8G8B8A8_UNORM.  For exact 2:1 levels the float box on byte/255 values stored
 *                                  with round-to-nearest equals the integer (a+b+c+d+2)>>2, which is what runs there.
 *                                  (The plug-in's default for UNORM encodings is the WIC scaler, which is NOT in the tree:
 *                                  parity with WIC is unpinned; this is DirectXTex's TEX_FILTER_FORCE_NON_WIC result.)
 *   itw_generate_mips_device_srgb  RGBA8 as R8G8B8A8_UNORM_SRGB: filtered in linear light (XMColorSRGBToRGB after the load,
 *                                  XMColorRGBToSRGB before the store, DirectXTexConvert.cpp:2669-2685, :2757-2775) -- what the
 *                                  plug-in gets for BC1/BC3/BC7 *_SRGB encodings (IntelPlugin.cpp:152-154; WIC is bypassed for
 *                                  sRGB formats, DirectXTexMipmaps.cpp:389-393).  itw_dds_encode_texture / _pixels use it for
 *                                  dxgi_format 72 / 78 / 99.
 *   itw_generate_mips_device_f16   RGBA16F, the BC6H save path (TEX_FILTER_FORCE_NON_WIC, IntelPlugin.cpp:2117-2127).
 * Bit-exact to those generator bodies (cut and compiled by oracle/build_ref_frontend.py), including their stale fourth tap
 * on wide power-of-two textures (csrc/mips_f16.cuh).  Outside the tree and therefore assumed: XMLoadUByteN4 = byte*(1/255),
 * XMStoreUByteN4 = round to nearest, the half conversions of DirectXMath 3.06, the C library's powf.
 * ------------------------------------------------------------------------------------------- */
/* Bytes of device scratch for the padded levels first_level..levels-1 of a w x h RGBA8 texture. */
size_t itw_mip_scratch_bytes(int width, int height, int levels, int first_level);
/* Build padded levels 1..levels-1 (and a padded copy of level 0 if its size is not a multiple of 4) in
 * `scratch` (device, >= itw_mip_scratch_bytes(w, h, levels, pad0 ? 0 : 1)) from the device surface
 * `level0` (width/height = the true texture size, any stride).  out[l] receives the padded surface of
 * level l (out[0] = *level0 when no padding is needed).  Enqueued on `cuda_stream`; returns 0 on success. */
int itw_generate_mips_device(const rgba_surface* level0, int levels, rgba_surface* out, uint8_t* scratch,
                             void* cuda_stream);
/* Same arguments, sRGB-correct RGBA8 chain / RGBA16F chain (8-byte texels: scratch needs TWICE itw_mip_scratch_bytes(...)). */
int itw_generate_mips_device_srgb(const rgba_surface* level0, int levels, rgba_surface* out, uint8_t* scratch,
                                  void* cuda_stream);
int itw_generate_mips_device_f16(const rgba_surface* level0, int levels, rgba_surface* out, uint8_t* scratch,
                                 void* cuda_stream);
/* The complete save path of one texture (IntelPlugin.cpp:2117-2171): `tops` = array_size HOST or
 * device surfaces holding level 0 only (RGBA8; RGBA16F for BC6H_UF16 / _SF16); mips are generated on the
 * GPU, every level is encoded, and the DDS file is written to `file` (host).  Returns the file size, 0 on
 * error. */
size_t itw_dds_encode_texture(const itw_dds_desc* desc, const rgba_surface* tops, const void* settings,
                              uint8_t* file, size_t capacity);

/* ---------------------------------------------------------------------------------------------
 * Section 5 -- decoders (SURVEY.md 8f-3): what the plug-in's preview obtains from
 * DirectX::Decompress (IntelPlugin.cpp:1051-1066; DirectXTex/DirectXTexCompress.cpp:358-468 ->
 * D3DXDecodeBC1/3/4U/5U/6HU/7, BC.cpp:897, BC4BC5.cpp:369-400, BC6HBC7.cpp:2879-2900).
 * `blocks` holds (width/4)*(height/4) blocks in raster order; dst->ptr is WRITTEN: RGBA8 texels
 * (4 B) for BC1/BC3/BC4/BC5/BC7 (BC4: r,0,0,255; BC5: r,g,0,255), RGBA16F texels (8 B, half bit
 * patterns, alpha = 1.0) for BC6H_UF16 / BC6H_SF16 (signed decode: D3DXDecodeBC6HS).  width/height multiples of 4; either side may be host or
 * device memory; synchronous.  BC7 and BC6H are exact by the format definition; BC1-BC5 equal
 * DirectXTex's float decoders rounded to nearest (csrc/decode.cuh).  Returns 0 on success.
 * ------------------------------------------------------------------------------------------- */
int itw_decode(int format, const uint8_t* blocks, const rgba_surface* dst);

/* ---------------------------------------------------------------------------------------------
 * Section 6 -- pixel-format front end and the image-level entry (SURVEY.md 8f-4): what the plug-in
 * does between Photoshop's buffer and CompressBlocks*:
 *   CopyDataForEncoding (IntelPlugin.cpp:85-181) -> ConvertToBC{,4or5,6}From{8,16,32}Bit (:291-433,
 *   :741-810) with the scalar rules of IntelPlugin.h:41-96; FlipXYChannelNormalMap (:1504-1546);
 *   NormalizeNormalMapChain (:1551-1612); DoPaddingToMultiplesOf4 (:892-928).
 * All of it is per-texel work, fused here into ONE bandwidth-bound pass (the padding is a
 * coordinate clamp), optionally followed by the encoder without leaving the GPU.
 * ------------------------------------------------------------------------------------------- */
typedef struct itw_pixel_source {  /* Photoshop's FormatRecord as the converters read it */
    const void* data;              /* interleaved: element (x, y, c) at row y, index x*planes + c   */
    int32_t width, height;         /* texels; need NOT be multiples of 4                            */
    int32_t planes;                /* channels per texel in `data`, 1..4 (hiPlane - loPlane + 1)    */
    int32_t depth;                 /* 8; 16 = Photoshop's 0..32768 integers; 32 = float, gamma 1.0   */
    int64_t row_bytes;             /* bytes between rows; 0 = tightly packed (the plug-in's case)    */
} itw_pixel_source;
enum {
    ITW_FRONT_HAS_ALPHA = 1,   /* plane 3 is alpha (else alpha = 255 / 1.0); needs planes == 4          */
    ITW_FRONT_GAMMA = 2,       /* 32-bit LDR only: v^(1/2.2) before the byte conversion (IntelPlugin.h:71) */
    ITW_FRONT_FLIP_X = 4,      /* normal maps: r = 255 - r   /  half(1 - r)                              */
    ITW_FRONT_FLIP_Y = 8,      /* normal maps: g = 255 - g   /  half(1 - g)                              */
    ITW_FRONT_NORMALIZE = 16   /* normal maps: rgb re-normalised around 128 (LDR) / to unit length (HDR) */
};
/* Convert `src` for encoding to `format` (ITW_FORMAT_*): BC6H -> RGBA16F texels, everything else ->
 * RGBA8; missing planes are 0 (BC4/BC5: a copy of plane 0).  dst->width/height must be the source
 * size or that size rounded up to multiples of 4 (edge texels are replicated).  Either side may be
 * host or device memory; synchronous.  Returns 0 on success. */
int itw_convert_pixels(int format, const itw_pixel_source* src, uint32_t flags, const rgba_surface* dst);
/* The image-level entry (the seam of CompressImageST, win32Threads.h:57-58, moved above the
 * conversion): convert + pad + encode in one call; `dst_blocks` receives ((w+3)/4)*((h+3)/4)
 * blocks.  `settings` as for itw_encode_device.  Returns 0 on success. */
int itw_encode_pixels(int format, const itw_pixel_source* src, uint32_t flags, const void* settings,
                      uint8_t* dst_blocks);

/* The plug-in's whole save path (IntelPlugin.cpp:2062-2171) in one call: `sources` = array_size pixel
 * sources (level 0 of a 2-D texture, or the faces of a cube map) of desc->width x desc->height texels.
 * CopyDataForEncoding + FlipXYChannelNormalMap -> mip chain (as itw_dds_encode_texture) ->
 * NormalizeNormalMapChain on EVERY level when ITW_FRONT_NORMALIZE is set (the plug-in normalises after
 * the chain exists, :2149-2152) -> pad -> encode -> DDS blob in `file` (host).  Returns the file size, 0 on
 * error. */
size_t itw_dds_encode_pixels(const itw_dds_desc* desc, const itw_pixel_source* sources, uint32_t flags,
                             const void* settings, uint8_t* file, size_t capacity);

/* The save dialog's "mip maps from layers" option (DoWriteDDS, IntelPlugin.cpp:2093-2145 -> CopyLayersIntoMipMaps,
 * :1749-1850): each document layer supplies one mip level by hand.  Level l is read from the top-left
 * max(1, W >> l) x max(1, H >> l) texels of layer l, one planar buffer per channel, as ReadLayerData delivers them. */
typedef struct itw_layer_source {  /* one document layer as CopyLayersIntoMipMaps reads it                      */
    const void* channels[3];       /* compositeChannelsList in order: planar, the composite's depth, document-sized */
    int32_t channel_count;         /* 1..3                                                                       */
    const void* alpha;             /* layerMask, else transparency; NULL = FillLayerDataToWhite                   */
    int64_t row_bytes;             /* bytes between rows of every plane; 0 = width * depth / 8                   */
} itw_layer_source;
/* itw_dds_encode_pixels for a 2-D texture (array_size 1, not a cube map) whose levels come from `layers`, in the
 * plug-in's order: convert the composite -> layer 0 overwrites level 0 -> FlipXYChannelNormalMap on level 0 -> mip
 * chain from level 0 -> layer l overwrites level l for 1 <= l < min(layer_count, mip_levels) (extra layers are
 * ignored; levels without a layer keep the generated texels) -> NormalizeNormalMapChain on every level -> pad ->
 * encode.  So levels 1 and up taken from layers are NOT flipped, and generated levels come from the flipped level 0.
 * Per texel (CopyFromLayerChannelIntoImage, :1694-1741): channel c goes to plane c with the composite's converters,
 * except that RGBA8 targets at depth 32 always take the v^(1/2.2) step (ITW_FRONT_GAMMA does not matter here);
 * planes c >= channel_count keep what they held.  Plane 3 is ALWAYS written: from `alpha` when ITW_FRONT_HAS_ALPHA
 * is set and `alpha` is not NULL, else from white (FillLayerDataToWhite, :1664-1689).  At depth 16 that white is
 * ConvertTo16Bit((unsigned8)255) = 15360, not 32768, so a level from a 16-bit layer without alpha has alpha 119
 * (RGBA8) or 0x3780 (RGBA16F) where the composite gives 255 / 0x3C00 -- the plug-in's behaviour, reproduced.
 * `flags` and `settings` as for itw_dds_encode_pixels; layer_count == 0 gives that function's file.  Every operand
 * may be in host or device memory; only the read rectangles are copied.  Synchronous.  Returns the file size, or 0
 * with an error text and `file` untouched when an argument is wrong (nothing is enqueued then). */
size_t itw_dds_encode_layers(const itw_dds_desc* desc, const itw_pixel_source* composite, const itw_layer_source* layers,
                             int layer_count, uint32_t flags, const void* settings, uint8_t* file, size_t capacity);

/* ---------------------------------------------------------------------------------------------
 * Section 7 -- row-sharded encode over several GPUs, one process per GPU (SURVEY.md 8e, config C4):
 * "images shard row-wise across the GPUs with a single NCCL all-gather of the packed output".
 * Band rule = the reference's thread split (win32Threads.cpp:217-230).  Every rank holds its rows of level 0
 * of an RGBA8 texture on its device; mips are made band-locally while a level's band is a whole number of block
 * rows, each band is encoded where it lies, ONE ncclAllGather moves the packed bands (plus the few KiB of raw
 * texels the tiny remaining levels are filtered from), and every rank ends up with the complete packed chain --
 * byte-identical to the single-GPU encode of the same texture.  NCCL is bound at run time (libnccl.so.2, or the
 * path in ITW_NCCL_LIB); with no communicator the same call runs on one GPU.
 * ------------------------------------------------------------------------------------------- */
typedef struct itw_shard_plan {
    int32_t  nranks, rank, levels;
    int32_t  band_levels;         /* leading levels whose row bands are whole block rows on every rank            */
    int32_t  band_y0, band_y1;    /* rows of level 0 owned by `rank`                                              */
    uint64_t slot_bytes;          /* per-rank payload of the all-gather (multiple of 16)                          */
    uint64_t chain_bytes;         /* the complete packed chain, levels 0..levels-1 back to back (= DDS payload)   */
    uint64_t level_offset[16];    /* of level l in the chain                                                      */
    uint64_t level_bytes[16];
    uint64_t send_offset[16];     /* of this rank's band of level l inside its slot (l < band_levels)             */
    uint64_t band_bytes[16];      /* one rank's band of level l; rank r's band sits at level_offset + r*band_bytes */
    uint64_t texel_offset;        /* raw texels of level band_levels-1 inside the slot ...                        */
    uint64_t texel_bytes;         /* ... 0 when every level is band-local                                         */
} itw_shard_plan;
/* Pure arithmetic (no CUDA call): the layout used by itw_encode_mip_chain_sharded.  width/height multiples of 4,
 * levels <= 16, height / nranks a multiple of 4 rows.  Returns 0 on success. */
int itw_shard_plan_make(int format, int width, int height, int levels, int nranks, int rank, itw_shard_plan* plan);
/* NCCL bootstrap: rank 0 obtains an id (ncclGetUniqueId), the host passes it to the other ranks by its own means
 * (MPI, a torch.distributed broadcast, a file), every rank calls itw_shard_init on the thread and device it encodes
 * with (ncclCommInitRank).  itw_shard_finalize destroys the calling thread's communicator. */
int itw_shard_unique_id(uint8_t id[128]);
int itw_shard_init(int rank, int nranks, const uint8_t id[128]);
void itw_shard_finalize(void);
/* band0 = this rank's rows [band_y0, band_y1) of level 0 (device memory, any 4-byte aligned stride; width x
 * (band_y1-band_y0)); chain = device buffer of plan.chain_bytes (16-byte aligned) that receives the COMPLETE packed
 * chain on every rank.  Everything is enqueued on `cuda_stream` (cudaStream_t as void*), nothing is synchronised;
 * the scratch belongs to the calling thread, so consecutive calls of one thread must use one stream (or be separated
 * by a synchronisation).  `settings` as for itw_encode_device.  Returns 0 on success. */
int itw_encode_mip_chain_sharded(int format, const rgba_surface* band0, int width, int height, int levels,
                                 const void* settings, uint8_t* chain, void* cuda_stream);

/* ---------------------------------------------------------------------------------------------
 * Section 8 -- decompress for display and the preview path: what the plug-in's options dialog runs on
 * every settings change (GetCompressedImageForPreview, IntelPlugin.cpp:933-1080): front end -> encode ->
 * DirectX::Decompress (DirectXTexCompress.cpp:358-468 -> _ConvertScanline -> _StoreScanline) into the
 * format the dialog shows.
 * ------------------------------------------------------------------------------------------- */
enum {
    ITW_TARGET_R32G32B32A32_FLOAT = 2,    /* 16 B per texel                                     */
    ITW_TARGET_R8G8B8A8_UNORM = 28,       /* 4 B per texel                                      */
    ITW_TARGET_R8G8B8A8_UNORM_SRGB = 29   /* 4 B per texel                                      */
};
/* DirectX::Decompress of `blocks` (ceil(width/4) * ceil(height/4) blocks in raster order) into `dst`
 * (width x height texels of `target_dxgi`; texels of ragged edge blocks outside the image are not written).
 * Pairs (dxgi_format -> target):
 *   71/77/83/98 (UNORM)      -> 28: the bytes of itw_decode;  -> 29: XMColorRGBToSRGB, then the UNORM8 store
 *   80 (BC4 UNORM)           -> 28 / 29: as above with red copied into green and blue, (r, r, r, 255): DirectXTex converts
 *                               an R format to an RGB one that way (itw_decode gives (r, 0, 0, 255))
 *   72/78/99 (_SRGB)         -> 28: XMColorSRGBToRGB, then the UNORM8 store;  -> 29: the plain bytes
 *   95/96 (BC6H UF16 / SF16) -> 28: half -> float -> saturate -> UNORM8;  -> 2: half -> float, alpha 1.0
 * Other pairs are rejected before anything is enqueued.  Either side may be host or device memory (device
 * operands: the ordering rule of CompressBlocks*); synchronous.  Returns 0 on success. */
int itw_decompress(int dxgi_format, const uint8_t* blocks, int width, int height, int target_dxgi,
                   const rgba_surface* dst);
/* GetCompressedImageForPreview in one call.  count == 1: a 2-D document; count == 6: six faces of equal size
 * (+X,-X,+Y,-Y,+Z,-Z) laid out as a 4w x 3h horizontal cross (cells without a face are zero texels, flipped /
 * normalised like the rest).  Front end (`flags` = ITW_FRONT_*) -> [cross] -> pad -> encode to `dxgi_format`
 * (`settings` as for itw_encode_device) -> display decompress into `display`, which must have the size of the
 * image or cross and the texels of the target: R32G32B32A32_FLOAT (16 B) for BC6H at sources[0].depth == 32,
 * R8G8B8A8_UNORM (4 B) otherwise.  At depth 32 BC1/BC3/BC7 are shown as their _SRGB formats, at depths 8 / 16
 * _SRGB formats are shown as UNORM (IntelPlugin.cpp:1024-1059).  *compressed_bytes (may be NULL) receives the
 * size of the encoded image.  Cube maps of BC6H_SF16 are rejected (the plug-in builds that cross as RGBA8).
 * Everything between the copy-in of the planes and the copy-out of the display stays on the device.  Either
 * side may be host or device memory; synchronous.  Returns 0 on success. */
int itw_preview_pixels(int dxgi_format, const itw_pixel_source* sources, int count, uint32_t flags,
                       const void* settings, const rgba_surface* display, size_t* compressed_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 9 -- the open path: what the plug-in does when it opens a block-compressed DDS file, split as it splits the work:
 *   DoReadStart    (IntelPlugin.cpp:2419-2612)  LoadFromDDSMemory -> IsAlphaAllOpaque -> layers / planes / depth -> Decompress
 *                                               to R8G8B8A8_UNORM[_SRGB] or R32G32B32A32_FLOAT
 *   DoReadContinue (IntelPlugin.cpp:2614-2742)  once per layer: zero a full-size interleaved buffer, copy one image into it
 * The formats are those of itw_dds_desc: BC1, BC3, BC4, BC5, BC6H UF16 / SF16, BC7 and the _SRGB forms.  BC2, uncompressed and
 * palettised files are rejected (section 13 opens the uncompressed files the plug-in reads without a conversion).
 * ------------------------------------------------------------------------------------------- */
typedef struct itw_dds_open_info {
    itw_dds_desc desc;        /* as itw_dds_read_header                                                                */
    int32_t has_alpha;        /* the plug-in's loadInfo.hasAlpha (:2468-2472): HasAlpha(format) && !IsAlphaAllOpaque() and not
                                 BC1, where IsAlphaAllOpaque checks every texel of every image (all mips of all items) for a
                                 decoded alpha below 0.99.  Taken before the cube-map override.                           */
    int32_t has_mips;         /* mip_levels > 1                                                                         */
    int32_t ask_user;         /* the plug-in would show its load dialog (:2481-2490, after the cube-map override)        */
    /* filled by itw_dds_open_layout: */
    int32_t layers;           /* the number of layers the host creates: 0 (a background image), 1, 6 (a cube map) or
                                 mip_levels (mips as layers) (:2507-2532)                                               */
    int32_t calls;            /* itw_dds_read_layer calls = max(1, layers)                                              */
    int32_t planes, depth;    /* 3 or 4 channels; 8 (bytes) or 32 (floats) bits per channel (:2591-2602)                */
    int32_t width, height;    /* every layer: the top level (or one cube face)                                          */
    int32_t target_dxgi;      /* the Decompress target: 28 R8G8B8A8_UNORM, 29 R8G8B8A8_UNORM_SRGB, 2 R32G32B32A32_FLOAT  */
} itw_dds_open_info;
/* the load dialog's two answers (:2477-2504), or the values a script supplies */
enum { ITW_OPEN_SEPARATE_ALPHA = 1, ITW_OPEN_MIPS = 2 };
/* Header + the alpha check on the GPU.  Fills desc, has_alpha, has_mips and ask_user; zeroes the layout fields.  A file of
 * array_size 6 (one cube map) is read as a cube map, as the plug-in does.  Returns 0 on success. */
int itw_dds_open(const uint8_t* file, size_t size, itw_dds_open_info* info);
/* The layout for the dialog's answers `options` (ITW_OPEN_*); pure arithmetic, no CUDA call.  Cube maps ignore both answers.
 * Returns 0 on success. */
int itw_dds_open_layout(itw_dds_open_info* info, uint32_t options);
/* One DoReadContinue: layer `call` (0 <= call < info->calls) into `dst`, `height` rows of `width` interleaved texels of `planes`
 * channels of `depth` bits, rows `row_bytes` apart (0 = tightly packed).  Reads cube face `call` (mip 0) of a cube map, mip `call`
 * of item 0 when mips are layers, the first image otherwise.  Every byte of the layer is written: the image is DirectX::Decompress'ed
 * (BC4 as (r, r, r, 255), BC6H with alpha 1.0) into the top-left corner, channels 0..planes-1 are copied (BC1's punch-through
 * alpha included), the rest of the layer is zero, and a cube map with has_alpha gets its last plane set to 255 / 1.0f.  `file` and
 * `dst` may each be host or device memory (device operands: the ordering rule of CompressBlocks*); synchronous.  Every argument is
 * checked before anything is enqueued (a truncated file, a file that does not match info->desc, a call out of range, row_bytes
 * too small, info not laid out): on failure dst is untouched.  Returns 0 on success. */
int itw_dds_read_layer(const uint8_t* file, size_t size, const itw_dds_open_info* info, int call, void* dst, int64_t row_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 10 -- cube maps from the document: the save dialog's two cube texture types, CUBEMAP_CROSSED and CUBEMAP_LAYERS
 * (IntelPlugin.cpp:44-65), through DoWriteDDS (:2062-2171) and GetCompressedImageForPreview (:933-1080), with the dialog's
 * "set mip level" option (IsCubeMapWithSetMipLevelOverride, :1172-1179).
 *   cross   ConvertToCubeMapFromCross (:1200-1265): six W x H cells of one document.  A horizontal 4x3 cross (doc width >= doc
 *           height) gives W = doc_width / 4, H = doc_height / 3; a vertical 3x4 cross gives W = doc_width / 3, H = doc_height / 4 and
 *           takes -Z from cell (1, 3), unrotated.  For a 1/3/7 _SRGB encoding with mip maps the document scratch is
 *           R8G8B8A8_UNORM_SRGB (:152-154) and the cube scratch R8G8B8A8_UNORM (:1240-1246), so CopyRectangle LINEARISES r, g, b of
 *           every cell (XMColorSRGBToRGB, then the UNORM8 store); otherwise the cells are copied as converted.
 *   layers  ConvertToCubeMapFromLayers (:1270-1416): face i starts all zero (InitializeCube) and is filled from the layer named
 *           +X, -X, +Y, -Y, +Z, -Z by the per-texel rules of itw_dds_encode_layers (channels c < channel_count, alpha from the
 *           layer when ITW_FRONT_HAS_ALPHA is set and `alpha` is not NULL, else white -- 119 / 0x3780 at depth 16 -- and RGBA8
 *           targets always gamma-correct 32-bit layers).  W x H = the document size.  A face with no layer stays zero.
 * The chain is filtered as the cube scratch is: R8G8B8A8_UNORM for every 8-bit format (_SRGB included), RGBA16F for BC6H.
 * ------------------------------------------------------------------------------------------- */
enum { ITW_CUBE_CROSS = 0, ITW_CUBE_LAYERS = 1 };
typedef struct itw_cube_options {
    uint32_t dxgi_format;  /* the plug-in's cube columns: 71/72 BC1, 77/78 BC3, 95 BC6H_UF16, 98/99 BC7 (BC4, BC5 and BC6H_SF16 are
                              refused: the plug-in offers no cube of them, or builds it as RGBA8)                                    */
    int32_t  source;       /* ITW_CUBE_CROSS: the document is the cross; ITW_CUBE_LAYERS: six face layers                          */
    int32_t  mip_maps;     /* 0 / 1: the dialog's MipMapTypeIndex != NONE (AUTOGEN or FROM_LAYERS: DoMipMaps, :2056)               */
    int32_t  mip_level;    /* -1, or L: the set mip level.  The file is then the one-level cube of level L of every face
                              (SaveCubeMipLevelToDDSFile, :1856-1871); 0 <= L < max(W, H).bit_length()                            */
} itw_cube_options;
/* Pure arithmetic, no CUDA call: the face size (*face_width / *face_height, may be NULL) and the desc of the file the save writes.
 * Without L: W x H, the full chain with mip_maps, else 1 level.  With L: max(1, W >> L) x max(1, H >> L), 1 level.  Always array_size 6,
 * is_cubemap 1.  Returns the file size; 0 with an error text when the options or the document size are refused (a cross smaller
 * than one texel per face). */
size_t itw_cube_layout(const itw_cube_options* o, int doc_width, int doc_height, itw_dds_desc* desc, int* face_width, int* face_height);
/* DoWriteDDS for the two cube types.  `document` = the composite: its texels are read only for ITW_CUBE_CROSS (`data` may be NULL for
 * ITW_CUBE_LAYERS, where it gives the size and the depth).  `faces` = six itw_layer_source in +X,-X,+Y,-Y,+Z,-Z order, channels[0] NULL
 * for a face without a layer of that name; ignored for a cross (may be NULL).  Each face layer is read whole: W x H planes of the
 * document's depth.  `flags`: ITW_FRONT_HAS_ALPHA and ITW_FRONT_GAMMA only (the plug-in flips and normalises normal maps only,
 * :2103, :2151).  With L only levels 0..L are built and only level L is encoded (the plug-in encodes the whole chain and keeps
 * level L; the bytes of level L are the same).  `settings` as for itw_encode_device.  Every operand may be host or device memory
 * (the ordering rule of CompressBlocks*); synchronous.  Returns the file size, or 0 with an error text and `file` untouched when an
 * argument is refused (nothing is enqueued then). */
size_t itw_dds_encode_cube(const itw_cube_options* o, const itw_pixel_source* document, const itw_layer_source* faces, uint32_t flags,
                           const void* settings, uint8_t* file, size_t capacity);
/* GetCompressedImageForPreview for the two cube types, with itw_preview_pixels' display rules (target, shown format).  A cross without
 * L is the 2-D preview of the whole document (:966 does not fire): itw_preview_pixels with count 1.  Otherwise the faces are built
 * as for a save but never linearised (the preview's CopyDataForEncoding passes DoMipMaps = false, :957), the chain runs to L when
 * set, and the horizontal cross of level L (4 wL x 3 hL, cells without a face zero, :1421-1501) is padded, encoded and decompressed
 * into `display`, which must have the size of the document (cross without L) or of that cross.  *compressed_bytes (may be NULL)
 * receives the size of the encoded image.  Rejections as for itw_dds_encode_cube; `display` is then untouched.  Returns 0 on success. */
int itw_preview_cube(const itw_cube_options* o, const itw_pixel_source* document, const itw_layer_source* faces, uint32_t flags,
                     const void* settings, const rgba_surface* display, size_t* compressed_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 11 -- the preview dialog: the compressed pane of "mip maps from layers" (GetCompressedImageForPreview with
 * IsMipMapsDefinedByLayer, IntelPlugin.cpp:986-993) and the dialog's view of a pane (FetchPreviewRGB, :487-739), which
 * PreviewDialog::updatePreviewBuffer (PreviewDialog.cpp:260-274) calls for both panes on every repaint, pan, zoom or channel toggle.
 * ------------------------------------------------------------------------------------------- */
/* itw_preview_pixels of a 2-D document whose level 0 comes from layer 0, in the plug-in's order: CopyDataForEncoding (no mip maps,
 * so the scratch is R8G8B8A8_UNORM even for _SRGB encodings) -> CopyLayersIntoMipMaps(..., 0, 1): layer 0 overwrites the converted
 * composite with the per-texel rules of itw_dds_encode_layers (white alpha when the layer has none -- 15360 at depth 16 -- and the
 * v^(1/2.2) step for 32-bit layers into RGBA8) -> FlipXYChannelNormalMap (so _SRGB encodings are flipped too, unlike the save path)
 * -> NormalizeNormalMapChain -> pad -> encode -> display decompress, with itw_preview_pixels' display rules (target, shown format).
 * `layer0` is read whole: composite->width x composite->height planes of the composite's depth.  *compressed_bytes (may be NULL)
 * receives the slice pitch of level 0.  Every operand may be host or device memory; synchronous.  Rejections (those of
 * itw_dds_encode_layers for layer 0 and of itw_preview_pixels) happen before anything is enqueued and leave `display` untouched.
 * Returns 0 on success. */
int itw_preview_layers(int dxgi_format, const itw_pixel_source* composite, const itw_layer_source* layer0, uint32_t flags,
                       const void* settings, const rgba_surface* display, size_t* compressed_bytes);

enum { ITW_VIEW_RED = 0x4, ITW_VIEW_GREEN = 0x8, ITW_VIEW_BLUE = 0x10, ITW_VIEW_ALPHA = 0x20 };   /* PREVIEW_CHANNEL_* values */
typedef struct itw_view {
    int32_t  width, height;   /* the dialog buffer: width*height packed RGB8 texels                                    */
    int32_t  x, y;            /* previewOffsetX / Y                                                                      */
    double   zoom;            /* what the dialog passes: 1.f / previewZoom                                               */
    int32_t  mip_level;       /* SetMipLevel ? MipLevel : 0; zoom is divided by 1 << mip_level as at :503-504            */
    uint32_t channels;        /* ITW_VIEW_* mask; 0 = RGB (:492-493)                                                    */
    uint32_t matte;           /* 0x00BBGGRR                                                                              */
} itw_view;
/* FetchPreviewRGB's sampling into `dst` (view->width * view->height * 3 bytes, rows tightly packed).  `source` is the document
 * (depth 8, 16 or 32, planes 1..4, any row_bytes) or a pane: the display of itw_preview_pixels / _layers / _cube as R8G8B8A8_UNORM
 * (depth 8, planes 4) or R32G32B32A32_FLOAT (depth 32, planes 4); the plug-in switches on depth and format together, so those share
 * the branches of depths 8 and 32.  Dialog texel (xt, yt) shows source texel (int((xt + x) * z), int((yt + y) * z)), z = zoom /
 * (1 << mip_level), in double and truncated toward zero (an offset in (-1, 0) lands on texel 0); texels outside the source get the
 * matte bytes.  Channels (:585-624): pure R, G, B or A show grey, in a mixture alpha takes the blue slot, a channel beyond `planes`
 * shows 0.  Stores: depth 8 the byte, depth 16 FloatToByte(v / 32768.0), depth 32 FloatToByte((double)f) without gamma.
 * The exposure is 1: the value InitData sets at every DoWriteStart (:1889, :1902), before the user moves the slider; section 18's
 * itw_preview_view_exposed takes the slider's value.  Not covered: the R16G16B16A16_FLOAT branch (no pane is built in that
 * format).  Either side may be host or device memory (a host source is copied whole; device operands: the
 * ordering rule of CompressBlocks*); synchronous.  Every argument is checked before anything is enqueued (null pointers, a depth,
 * planes or row_bytes the source cannot have, a non-positive view size, a zoom that is not positive and finite, mip_level outside
 * 0..30, channel bits other than ITW_VIEW_*): `dst` is then untouched.  Returns 0 on success. */
int itw_preview_view(const itw_pixel_source* source, const itw_view* view, uint8_t* dst);

/* GetUncompressedImageForPreview (IntelPlugin.cpp:1085-1167): the original pane when the mip-map type is FROM_LAYERS or the texture
 * type is a cube type (FetchPreviewRGB, :565-580), and the compressed pane of the "none" encoding, which the dialog takes from this
 * function because GetCompressedImageForPreview returns NULL for it (:936-941, :551-552).  Every encoding but BC6H_UF16 gives an
 * R8G8B8A8_UNORM scratch, so the pane is built in the plug-in's order with no DirectX::Convert:
 *   CopyDataForEncoding(DoMipMaps = false, gammaCorrect = false): the ConvertToBC4or5From* front end for 80 / 83, ConvertToBCFrom*
 *       for every other encoding (28 included); no _SRGB scratch, and depth 32 WITHOUT the v^(1/2.2) step
 *   cube types (:1105-1121): the faces as itw_preview_cube builds them (never linearised), the chain to L when set, and the zeroed
 *       horizontal cross of level L (4 wL x 3 hL).  A cross without L is the converted document, as for ITW_PANE_2D
 *   mip maps from layers: layer 0 over the converted document (CopyLayersIntoMipMaps(..., 0, 1)) with the per-texel rules of
 *       itw_dds_encode_layers: white alpha when the layer has none (15360 at depth 16) and the v^(1/2.2) step for 32-bit layers
 *   FlipXYChannelNormalMap (:1137-1140), after layer 0
 * and nothing else: no normalisation, padding, encode or decode.  The pane depends on the encoding only through its front end, so
 * 28, 71, 72, 77, 78, 98 and 99 give one pane. */
enum { ITW_PANE_2D = 0, ITW_PANE_CUBE_CROSS = 1, ITW_PANE_CUBE_LAYERS = 2 };
typedef struct itw_pane_options {
    uint32_t dxgi_format;  /* the dialog's encoding: 71/72 BC1, 77/78 BC3, 80 BC4, 83 BC5, 98/99 BC7 or 28 (none, R8G8B8A8_UNORM).
                              95 is refused here (section 18's itw_preview_uncompressed_hdr builds its pane), 96 and every
                              other id too                                                                                       */
    int32_t  texture;      /* ITW_PANE_2D (COLOR, COLOR+A, NORMAL MAP) or one of the two cube types                            */
    int32_t  mip_level;    /* cube types: the set mip level (SetMipLevel ? MipLevel : -1), -1 <= L < max(W, H).bit_length() of
                              the face; ITW_PANE_2D: must be -1                                                                  */
} itw_pane_options;
/* The pane into `display` (R8G8B8A8_UNORM: 4-byte texels, rows `stride` >= 4 * width bytes apart).  `display` has the size of the
 * document (ITW_PANE_2D, or a cross without L) or of the cross of level L.  A device display that is 4-byte aligned (pointer and
 * stride) is written in place, so itw_preview_view can sample it with no copy; a host display receives one device-to-host copy.
 * `layers`: ITW_PANE_2D: NULL, or layer 0 when the host's IsMipMapsDefinedByLayer() holds (read whole, document-sized planes of the
 * document's depth); ITW_PANE_CUBE_LAYERS: six faces +X,-X,+Y,-Y,+Z,-Z as for itw_dds_encode_cube (channels[0] NULL for a face
 * without a layer); ITW_PANE_CUBE_CROSS: ignored.  `flags`: ITW_FRONT_HAS_ALPHA (the plug-in's planes > 3), and ITW_FRONT_FLIP_X /
 * _Y for ITW_PANE_2D only; ITW_FRONT_GAMMA and ITW_FRONT_NORMALIZE are refused (the pane never takes either step).
 * *compressed_bytes (may be NULL) receives the dialog's compressed size: width * height * 4 of the DOCUMENT for 28 (also for the
 * cube types, whose pane is the larger cross, :939), 0 for the other encodings.  Every operand may be host or device memory (device
 * operands: the ordering rule of CompressBlocks*); synchronous; itw_last_kernel_ms gives the time of the call's kernels.  Every
 * argument is checked before anything is enqueued (those itw_preview_layers and itw_preview_cube check, the encoding, BC4 / BC5 with
 * a cube type, flags, a set level for ITW_PANE_2D): `display` is then untouched.  Returns 0 on success. */
int itw_preview_uncompressed(const itw_pane_options* o, const itw_pixel_source* document, const itw_layer_source* layers,
                             uint32_t flags, const rgba_surface* display, size_t* compressed_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 12 -- saving the "none" encoding: the uncompressed R8G8B8A8_UNORM (DXGI 28) DDS file that DoWriteDDS writes when the
 * dialog's encoding is "none" (IntelPlugin.cpp:2051-2194), for every texture type the dialog allows it with (COLOR, COLOR+A, NORMAL
 * MAP and both cube types, IsCombinationValid :44-65).  The steps are those of the other saves, in the plug-in's order:
 *   CopyDataForEncoding(DoMipMaps, gammaCorrect = true): the ConvertToBCFrom* front end (:147-177), the v^(1/2.2) step at depth 32
 *       with ITW_FRONT_GAMMA; the scratch is always R8G8B8A8_UNORM (28 is not sRGB, so there is no _SRGB scratch)
 *   cube types: the faces of itw_dds_encode_cube (never linearised), the chain to L with a set level
 *   2-D: layer 0 over level 0 (mip maps from layers), FlipXYChannelNormalMap, the chain, layers 1.. into their levels,
 *       NormalizeNormalMapChain on every level
 * and then no encode (CompressToScratchImage swaps the scratch in, :262-268): SaveToDDSMemory (or SaveCubeMipLevelToDDSFile, :1856-1871,
 * for a set level) writes every level as it is, rows of 4 * w_l bytes with no padding, item-major and mip-minor, behind the legacy
 * 128-byte header of _EncodeDDSHeader (DDSPF_A8B8G8R8, DDS_HEADER_FLAGS_PITCH, pitch 4 * width; one cube of six faces stays legacy).
 * The chain is DirectXTex's non-WIC generators (box for power-of-two sizes, else linear), as for every UNORM save here; the plug-in's
 * GenerateMipMaps hands R8G8B8A8_UNORM to WIC, which is not in the tree, so parity with WIC's filters is not pinned.
 * Format 28 stays unknown to every other call of this header (itw_dds_header_bytes, itw_dds_write_header, itw_dds_open, ...); section 13
 * opens these files.
 * ------------------------------------------------------------------------------------------- */
typedef struct itw_none_options {
    int32_t texture;       /* ITW_PANE_2D (COLOR, COLOR+A, NORMAL MAP), ITW_PANE_CUBE_CROSS or ITW_PANE_CUBE_LAYERS                    */
    int32_t mip_maps;      /* 0 / 1: the dialog's DoMipMaps (mip-map type AUTOGEN or FROM_LAYERS)                                     */
    int32_t mip_level;     /* cube types: -1, or the set mip level L with the bound of itw_cube_layout; ITW_PANE_2D: must be -1         */
} itw_none_options;
/* Pure arithmetic, no CUDA call: the desc of the file (dxgi_format 28) and the level-0 size of an item (*face_width / *face_height:
 * the document for ITW_PANE_2D, the face for the cube types; each may be NULL).  ITW_PANE_2D: the document, the full chain
 * (max(W, H).bit_length() levels) with mip_maps, else one level.  Cube types: as itw_cube_layout.  Returns the file size, 128 +
 * the sum over items and levels of 4 * w_l * h_l; 0 with an error text when refused. */
size_t itw_dds_none_layout(const itw_none_options* o, int doc_width, int doc_height, itw_dds_desc* desc, int* face_width, int* face_height);
/* DoWriteDDS with the "none" encoding into `file` (capacity >= the size itw_dds_none_layout gives).
 * ITW_PANE_2D: `document` is the composite; `layers` / `layer_count` as for itw_dds_encode_layers (layer_count 0 when the host's
 * IsMipMapsDefinedByLayer() is false); every ITW_FRONT_* flag applies.  Cube types: `document` and `layers` (the six faces, layer_count
 * 6; ignored for a cross) as for itw_dds_encode_cube; only ITW_FRONT_HAS_ALPHA and ITW_FRONT_GAMMA apply.  Every operand may be host
 * or device memory (device operands: the ordering rule of CompressBlocks*); synchronous; itw_last_kernel_ms gives the time of the
 * call's kernels.  Every argument is checked before anything is enqueued (those of itw_dds_encode_layers and itw_dds_encode_cube,
 * the options, layer_count, the file and its capacity): `file` is then untouched.  Returns the file size, or 0 with an error text
 * that starts with the call's name. */
size_t itw_dds_save_none(const itw_none_options* o, const itw_pixel_source* document, const itw_layer_source* layers, int layer_count,
                         uint32_t flags, uint8_t* file, size_t capacity);

/* ---------------------------------------------------------------------------------------------
 * Section 13 -- opening uncompressed files: the DDS files whose loaded format (LoadFromDDSMemory with DDS_FLAGS_NONE, the header
 * rules of _DecodeDDSHeader / _GetDXGIFormat, DirectXTexDDS.cpp:144-437) is already DoReadStart's target (IntelPlugin.cpp:2534-2553),
 * so the plug-in runs neither Decompress nor Convert:
 *   28 R8G8B8A8_UNORM       -> depth 8        29 R8G8B8A8_UNORM_SRGB -> depth 8
 *   11 R16G16B16A16_UNORM   -> depth 16       2 R32G32B32A32_FLOAT   -> depth 32
 * The files of itw_dds_save_none are among them.  The header forms accepted (ITW_RAW_*) are a 'DX10' header naming 2, 11, 28 or 29,
 * and the legacy pixel formats that load as one of them.  A legacy header is matched as _GetDXGIFormat matches it: the first entry
 * of g_LegacyDDSMap whose flags intersect the header's and whose FourCC (FourCC entries), bit count (palette entries) or bit count
 * and four masks (the others) are equal.  Refused, with a message naming the call and the reason: every file whose loaded format
 * differs from its target (A8R8G8B8 / X8R8G8B8 load as B8G8R8A8 / B8G8R8X8, 565, 5551, 4444, L8, L16, A8L8, A8, G16R16, 10:10:10:2,
 * FourCC 113 and the other float FourCCs, DX10 ids other than the four above: the plug-in converts them with DirectX::Convert, which
 * can hand them to WIC), the palettised and 3:3:2 / 4:4 expansions (P8, A8P8, A8R3G3B2, R3G3B2, A4L4), block-compressed files (use
 * itw_dds_open), volumes, arrays other than one cube map, partial cubes, truncated files, width or height 0 or above 16777216.
 * The shapes are those of itw_dds_open: a 2-D texture with or without a mip chain, or one cube map (six faces).
 * ------------------------------------------------------------------------------------------- */
enum {
    ITW_RAW_DX10 = 0,        /* 'DX10' extension header naming 2, 11, 28 or 29 (payload at 148)                                  */
    ITW_RAW_A8B8G8R8 = 1,    /* DDSPF_A8B8G8R8 -> 28 (the header of itw_dds_save_none)                                           */
    ITW_RAW_X8B8G8R8 = 2,    /* DDSPF_X8B8G8R8 -> 28 with alpha 255 (CONV_FLAGS_NOALPHA)                                         */
    ITW_RAW_R8G8B8 = 3,      /* DDSPF_R8G8B8, 24 bpp -> 28: rows of 3 w bytes, texels stored B, G, R, alpha 255 (CONV_FLAGS_888)  */
    ITW_RAW_A16B16G16R16 = 4,/* FourCC 36 -> 11                                                                                  */
    ITW_RAW_A32B32G32R32F = 5/* FourCC 116 -> 2                                                                                  */
};
typedef struct itw_dds_uncompressed_info {
    itw_dds_desc desc;        /* width, height, mip_levels, array_size (1 or 6), is_cubemap; dxgi_format = the loaded format:
                                 2, 11, 28 or 29 (unknown to the calls of section 3, which keep refusing these formats)          */
    int32_t source;           /* ITW_RAW_*: the header form                                                                     */
    uint64_t payload_offset;  /* where the payload starts in the file: 128, or 148 behind a 'DX10' header                         */
    int32_t has_alpha;        /* loadInfo.hasAlpha: !IsAlphaAllOpaque() over every texel of every image (alpha < 0.99f); always 0
                                 for X8B8G8R8 and R8G8B8, whose alpha the loader sets to 255.  Taken before the cube-map override  */
    int32_t has_mips, ask_user;   /* as in itw_dds_open_info                                                                     */
    /* filled by itw_dds_uncompressed_layout, with the meanings of itw_dds_open_info: */
    int32_t layers, calls, planes;
    int32_t depth;            /* 8 (bytes), 16 (ushorts) or 32 (floats) bits per channel                                         */
    int32_t width, height;
    int32_t target_dxgi;      /* the loaded format, which is the target: 2, 11, 28 or 29                                         */
} itw_dds_uncompressed_info;
/* Header + the alpha check on the GPU.  Fills desc, source, payload_offset, has_alpha, has_mips and ask_user; zeroes the layout
 * fields.  A device-resident file is scanned where it lies; a host file's payload is copied to the device once.  Synchronous;
 * itw_last_kernel_ms gives the scan's time (-1 when the form needs no scan).  Returns 0 on success; on failure `info` is untouched. */
int itw_dds_open_uncompressed(const uint8_t* file, size_t size, itw_dds_uncompressed_info* info);
/* The layout for the dialog's answers `options` (ITW_OPEN_*), with itw_dds_open_layout's decisions; pure arithmetic, no CUDA call.
 * Returns 0 on success. */
int itw_dds_uncompressed_layout(itw_dds_uncompressed_info* info, uint32_t options);
/* One DoReadContinue, with the image choice, the zeroed layer and the rules of itw_dds_read_layer: channels 0..planes-1 of the loaded
 * texel (R8G8B8 and X8B8G8R8 expanded with alpha 255), and for a cube map with has_alpha the last plane forced to 255 (depth 8), 1.0f
 * (depth 32) or 0x3C00 (depth 16: the plug-in's ConvertTo16Bit((unsigned8)255), a half-float 1.0 in a UNORM16 plane).  16-bit
 * planes receive the file's 0..65535 values unscaled, as the plug-in hands them to Photoshop.  `file` and `dst` may each be host or
 * device memory (device operands: the ordering rule of CompressBlocks*); synchronous.  Every argument is checked before anything is
 * enqueued: on failure dst is untouched.  Returns 0 on success. */
int itw_dds_read_uncompressed_layer(const uint8_t* file, size_t size, const itw_dds_uncompressed_info* info, int call, void* dst,
                                    int64_t row_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 14 -- opening converted files: the uncompressed DDS files whose loaded format DoReadStart converts with DirectX::Convert
 * (IntelPlugin.cpp:2534-2560, filter 0) and for which _UseWICConversion (DirectXTexConvert.cpp:4161-4266) chooses the non-WIC _Convert:
 * _LoadScanline, _ConvertScanline, _StoreScanline per texel.  Loaded format -> target / depth:
 *   10 R16G16B16A16_FLOAT, 54 R16_FLOAT, 34 R16G16_FLOAT, 13 R16G16B16A16_SNORM, 35 R16G16_UNORM, 37 R16G16_SNORM, 58 R16_SNORM,
 *   26 R11G11B10_FLOAT, 67 R9G9B9E5_SHAREDEXP                              -> 11 R16G16B16A16_UNORM, depth 16
 *   49 R8G8_UNORM, 51 R8G8_SNORM, 31 R8G8B8A8_SNORM, 63 R8_SNORM, 65 A8_UNORM, 115 B4G4R4A4_UNORM -> 28 R8G8B8A8_UNORM, depth 8
 *   16 R32G32_FLOAT                                                        -> 2 R32G32B32A32_FLOAT, depth 32
 * SNORM channels become v * 0.5 + 0.5, FLOAT channels are saturated into UNORM targets, absent channels are 0 (alpha 1), and the
 * one-channel formats R16_FLOAT, R16_SNORM and R8_SNORM are replicated into red, green and blue.  A8L8 loads as R8G8 (L in red, A in
 * green, as DirectXTex loads it).  Refused, each with a message naming the call: the files Convert hands to WIC (A8R8G8B8 / X8R8G8B8
 * and the other B8G8R8A8 / B8G8R8X8 forms, 565, 5551, 10:10:10:2, XR_BIAS, L8, L16, R32F, D32_FLOAT, D16_UNORM), R32G32B32_FLOAT
 * (whose WIC use depends on the runtime), the four formats of section 13 (use itw_dds_open_uncompressed), block-compressed files (use
 * itw_dds_open), UINT / SINT / typeless / other depth / video formats, RGBG / GRGB / YUY2 / UYVY, the palettised and 3:3:2 / 4:4 expansions, volumes, arrays other
 * than one cube map, partial cubes and truncated files.  Shapes and rules are those of section 13.
 * ------------------------------------------------------------------------------------------- */
enum {
    ITW_CONV_DX10 = 0,            /* 'DX10' extension header naming one of the loaded formats above (payload at 148)               */
    ITW_CONV_G16R16 = 1,          /* D3DFMT_G16R16 -> 35                                                                          */
    ITW_CONV_A8L8 = 2,            /* D3DFMT_A8L8 -> 49                                                                            */
    ITW_CONV_A8 = 3,              /* D3DFMT_A8 -> 65                                                                              */
    ITW_CONV_A4R4G4B4 = 4,        /* D3DFMT_A4R4G4B4 -> 115                                                                       */
    ITW_CONV_X4R4G4B4 = 5,        /* D3DFMT_X4R4G4B4 -> 115 with the alpha nibble set to 0xF (CONV_FLAGS_NOALPHA)                  */
    ITW_CONV_Q16W16V16U16 = 6,    /* FourCC 110 -> 13                                                                             */
    ITW_CONV_R16F = 7,            /* FourCC 111 -> 54                                                                             */
    ITW_CONV_G16R16F = 8,         /* FourCC 112 -> 34                                                                             */
    ITW_CONV_A16B16G16R16F = 9,   /* FourCC 113 -> 10                                                                             */
    ITW_CONV_G32R32F = 10         /* FourCC 115 -> 16                                                                             */
};
typedef struct itw_dds_converted_info {
    itw_dds_desc desc;        /* width, height, mip_levels, array_size (1 or 6), is_cubemap; dxgi_format = the loaded format       */
    int32_t form;             /* ITW_CONV_*: the header form                                                                    */
    uint64_t payload_offset;  /* where the payload starts in the file: 128, or 148 behind a 'DX10' header                         */
    int32_t has_alpha;        /* loadInfo.hasAlpha: HasAlpha(loaded) && !IsAlphaAllOpaque() (alpha < 0.99f, read as the loaded
                                 format); always 0 for the formats without alpha and for X4R4G4B4.  Taken before the cube override */
    int32_t has_mips, ask_user;   /* as in itw_dds_open_info                                                                     */
    /* filled by itw_dds_converted_layout, with the meanings of itw_dds_open_info: */
    int32_t layers, calls, planes;
    int32_t depth;            /* 8 (bytes), 16 (ushorts) or 32 (floats) bits per channel                                         */
    int32_t width, height;
    int32_t target_dxgi;      /* the target: 2, 11 or 28                                                                         */
} itw_dds_converted_info;
/* Header + the alpha check on the GPU, as itw_dds_open_uncompressed.  itw_last_kernel_ms gives the scan's time (-1 when the format has
 * no alpha).  Returns 0 on success; on failure `info` is untouched. */
int itw_dds_open_converted(const uint8_t* file, size_t size, itw_dds_converted_info* info);
/* The layout for the dialog's answers `options` (ITW_OPEN_*); pure arithmetic, no CUDA call.  Returns 0 on success. */
int itw_dds_converted_layout(itw_dds_converted_info* info, uint32_t options);
/* One DoReadContinue: the image the call reads, converted texel by texel into the target and stored into the zeroed layer, with the
 * rules of itw_dds_read_uncompressed_layer (cube alpha forcing, 16-bit planes unscaled, host or device operands, every argument
 * checked before anything is enqueued).  Returns 0 on success. */
int itw_dds_read_converted_layer(const uint8_t* file, size_t size, const itw_dds_converted_info* info, int call, void* dst,
                                 int64_t row_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 15 -- opening the other block-compressed files: the ones itw_dds_open does not serve, which DoReadStart decompresses with
 * DirectX::Decompress (_DecompressBC, DirectXTexCompress.cpp:358-468, after its promotion of the typeless formats) as it does the
 * formats of section 9.  Loaded format (header forms) -> decoder -> target / depth:
 *   74 BC2_UNORM ('DX10', DXT3, DXT2), 73 BC2_TYPELESS        -> D3DXDecodeBC2                       -> 28 R8G8B8A8_UNORM, depth 8
 *   75 BC2_UNORM_SRGB                                          -> D3DXDecodeBC2                       -> 29 R8G8B8A8_UNORM_SRGB, depth 8
 *   77 BC3_UNORM (DXT4 only), 76 BC3_TYPELESS                  -> D3DXDecodeBC3                       -> 28, depth 8
 *   70 BC1_TYPELESS                                            -> D3DXDecodeBC1                       -> 28, depth 8
 *   79 BC4_TYPELESS, 82 BC5_TYPELESS                           -> BC4U / BC5U, red copied into g, b   -> 28, depth 8 (BC4)
 *   81 BC4_SNORM ('DX10', BC4S)                                -> D3DXDecodeBC4S, v * 0.5 + 0.5, red into green and blue -> 28
 *   84 BC5_SNORM ('DX10', BC5S)                                -> D3DXDecodeBC5S, v * 0.5 + 0.5 (blue 0 -> 128) -> 28
 *   94 BC6H_TYPELESS                                           -> BC6H_UF16, saturated               -> 11 R16G16B16A16_UNORM, depth 16
 *   97 BC7_TYPELESS                                            -> D3DXDecodeBC7                       -> 28, depth 8
 * has_alpha is HasAlpha(loaded) && !IsAlphaAllOpaque() for 70, 73-77 and 97, and the plug-in's BC1 exclusion names only 71 / 72, so a
 * BC1_TYPELESS file with punch-through texels opens with alpha.  Colours of DXT2 / DXT4 files reach the layers still premultiplied,
 * as in the plug-in.  Refused, each with a message naming the call: the formats and forms itw_dds_open serves (use itw_dds_open),
 * uncompressed files (use itw_dds_open_uncompressed or itw_dds_open_converted), the palettised and 3:3:2 / 4:4 expansions, volumes,
 * arrays other than one cube map, partial cubes, truncated files and zero or oversized dimensions.  Shapes and rules are those of
 * section 13.
 * ------------------------------------------------------------------------------------------- */
enum {
    ITW_OBC_DX10 = 0,       /* 'DX10' extension header naming one of the loaded formats above except 77 (payload at 148)            */
    ITW_OBC_DXT3 = 1,       /* FourCC DXT3 -> 74                                                                                   */
    ITW_OBC_DXT2 = 2,       /* FourCC DXT2 -> 74 (premultiplied alpha)                                                              */
    ITW_OBC_DXT4 = 3,       /* FourCC DXT4 -> 77 (premultiplied alpha)                                                              */
    ITW_OBC_BC4S = 4,       /* FourCC BC4S -> 81                                                                                   */
    ITW_OBC_BC5S = 5        /* FourCC BC5S -> 84                                                                                   */
};
typedef struct itw_dds_other_bc_info {
    itw_dds_desc desc;        /* width, height, mip_levels, array_size (1 or 6), is_cubemap; dxgi_format = the loaded format       */
    int32_t form;             /* ITW_OBC_*: the header form                                                                     */
    uint64_t payload_offset;  /* where the payload starts in the file: 128, or 148 behind a 'DX10' header                         */
    int32_t has_alpha;        /* loadInfo.hasAlpha: HasAlpha(loaded) && !IsAlphaAllOpaque() (alpha < 0.99f in a texel of any image);
                                 always 0 for 79, 81, 82, 84 and 94.  Taken before the cube override                              */
    int32_t has_mips, ask_user;   /* as in itw_dds_open_info                                                                     */
    /* filled by itw_dds_other_bc_layout, with the meanings of itw_dds_open_info: */
    int32_t layers, calls, planes;
    int32_t depth;            /* 8 (bytes) or 16 (ushorts, BC6H_TYPELESS) bits per channel                                        */
    int32_t width, height;
    int32_t target_dxgi;      /* the target: 28, 29 or 11                                                                        */
} itw_dds_other_bc_info;
/* Header + the alpha check on the GPU (open_alpha_kernel over every image), as itw_dds_open.  itw_last_kernel_ms gives the scan's time
 * (-1 when the format has no alpha).  Returns 0 on success; on failure `info` is untouched. */
int itw_dds_open_other_bc(const uint8_t* file, size_t size, itw_dds_other_bc_info* info);
/* The layout for the dialog's answers `options` (ITW_OPEN_*); pure arithmetic, no CUDA call.  Returns 0 on success. */
int itw_dds_other_bc_layout(itw_dds_other_bc_info* info, uint32_t options);
/* One DoReadContinue: the image the call reads, decompressed into the target and stored into the zeroed layer, with the rules of
 * itw_dds_read_uncompressed_layer (cube alpha forcing, host or device operands, every argument checked before anything is enqueued).
 * Returns 0 on success. */
int itw_dds_read_other_bc_layer(const uint8_t* file, size_t size, const itw_dds_other_bc_info* info, int call, void* dst,
                                int64_t row_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 16 -- opening palettised and legacy-expanded files: the D3D9-era pixel formats that LoadFromDDSMemory (DDS_FLAGS_NONE)
 * expands while it loads (CONV_FLAGS_EXPAND, _LegacyExpandScanline, DirectXTexDDS.cpp:726-1018).  Header form -> loaded format ->
 * target / depth:
 *   P8        (DDS_PAL8, 8 bits)                 -> 28 R8G8B8A8_UNORM: the palette entry of the index        -> 28, depth 8
 *   A8P8      (DDS_PAL8, 16 bits)                -> 28: the entry of the low byte, its alpha OR'd with the high byte -> 28
 *   A8R3G3B2  (RGB, 16 bits, e0 / 1c / 03 / ff00) -> 28: each 3- / 2-bit field bit-replicated, alpha the high byte -> 28
 *   A4L4      (LUMINANCE, 8 bits, 0f / - / - / f0) -> 115 B4G4R4A4_UNORM (l | l << 4 | l << 8 | a << 12), then DirectX::Convert's
 *                                                   non-WIC _Convert into 28, as section 14 converts A4R4G4B4           -> 28
 * A palettised file holds its 256 palette words (R, G, B, and a fourth byte that is the alpha: D3D9's peFlags) between the header
 * and the payload, so its payload starts at 1152.  A P8 file whose palette has 0 in that byte opens with transparent layers, as in
 * the plug-in.  has_alpha is IsAlphaAllOpaque on the loaded format over every texel of every image; a palette entry no texel uses
 * never counts.  Refused, each with a message naming the call: R3G3B2 (it loads as B5G6R5_UNORM, which Convert hands to WIC),
 * the files the calls of sections 9, 13, 14 and 15 serve (the message names the call), 'DX10' headers naming 113 (P8) or 114 (A8P8),
 * which LoadFromDDSMemory itself refuses, every other 'DX10' header, files that end inside the palette, truncated payloads, volumes,
 * arrays, partial cubes and zero or oversized dimensions.  Shapes and rules are those of section 13.
 * ------------------------------------------------------------------------------------------- */
enum {
    ITW_EXP_P8 = 0,           /* DDS_PAL8, 8 bits -> 28 (palette at 128, payload at 1152)                                         */
    ITW_EXP_A8P8 = 1,         /* DDS_PAL8, 16 bits -> 28 (palette at 128, payload at 1152)                                        */
    ITW_EXP_A8R3G3B2 = 2,     /* DDS_RGB, 16 bits, masks e0 / 1c / 03 / ff00 -> 28                                                */
    ITW_EXP_A4L4 = 3          /* DDS_LUMINANCE, 8 bits, masks 0f / 0 / 0 / f0 -> 115                                              */
};
typedef struct itw_dds_expanded_info {
    itw_dds_desc desc;        /* width, height, mip_levels, array_size (1 or 6), is_cubemap; dxgi_format = the loaded format:
                                 28, or 115 for A4L4                                                                              */
    int32_t form;             /* ITW_EXP_*: the header form                                                                     */
    uint64_t payload_offset;  /* where the payload starts in the file: 1152 behind a palette, else 128                            */
    int32_t has_alpha;        /* loadInfo.hasAlpha: !IsAlphaAllOpaque() of the loaded texels (alpha < 0.99f in a texel of any
                                 image).  Taken before the cube override                                                        */
    int32_t has_mips, ask_user;   /* as in itw_dds_open_info                                                                     */
    /* filled by itw_dds_expanded_layout, with the meanings of itw_dds_open_info: */
    int32_t layers, calls, planes;
    int32_t depth;            /* 8: bytes                                                                                        */
    int32_t width, height;
    int32_t target_dxgi;      /* the target: 28                                                                                  */
} itw_dds_expanded_info;
/* Header + the alpha check on the GPU, as itw_dds_open_uncompressed; the palette reaches the scan by value.  itw_last_kernel_ms gives
 * the scan's time.  Returns 0 on success; on failure `info` is untouched. */
int itw_dds_open_expanded(const uint8_t* file, size_t size, itw_dds_expanded_info* info);
/* The layout for the dialog's answers `options` (ITW_OPEN_*); pure arithmetic, no CUDA call.  Returns 0 on success. */
int itw_dds_expanded_layout(itw_dds_expanded_info* info, uint32_t options);
/* One DoReadContinue: the image the call reads, expanded (and for A4L4 converted) texel by texel into the target and stored into the
 * zeroed layer, with the rules of itw_dds_read_uncompressed_layer (cube alpha forcing, host or device operands, every argument checked
 * before anything is enqueued).  Returns 0 on success. */
int itw_dds_read_expanded_layer(const uint8_t* file, size_t size, const itw_dds_expanded_info* info, int call, void* dst,
                                int64_t row_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 17 -- opening volume textures, 1-D textures and texture arrays: the shapes the calls of sections 9 and 13-16 refuse, in
 * every format those calls serve.  LoadFromDDSMemory loads the whole resource (_DecodeDDSHeader's dimension branches,
 * ScratchImage::Initialize, DirectXTexDDS.cpp:199-353, DirectXTexImage.cpp:257-301), and DoReadStart / DoReadContinue never look at
 * the dimension, so the plug-in opens:
 *   a volume (a legacy header with DDS_HEADER_FLAGS_VOLUME, which takes precedence over the cube caps, or 'DX10' dimension 4 with that
 *     flag and an array size of 1): dwDepth slices at level 0, halving per level, stored level-major; up to _CountMips3D levels.
 *     Each call reads slice 0 of its level (GetImage(mip, 0, 0)).
 *   a 1-D texture or 1-D array ('DX10' dimension 2): height 1 (a DDS_HEIGHT header must say 1), the cube flag dropped, up to
 *     _CountMips(w, 1) levels.
 *   a 2-D array or cube array ('DX10' dimension 3) of more than one item, for the formats of sections 13-16 (itw_dds_open serves the
 *     arrays of its formats).
 * An array_size of exactly 6 is read as a cube map whatever its dimension or cube flag (IntelPlugin.cpp:2479): six layers of item i,
 * mip 0, alpha forced when has_alpha is set.  Otherwise the calls read GetImage(call, 0, 0) when mips are layers, or the first image.
 * has_alpha is the serving section's: HasAlpha(loaded) && !IsAlphaAllOpaque() over EVERY image (every item, level and slice), so a
 * volume whose only translucent texels lie in slices no layer shows opens with has_alpha = 1, as in the plug-in.  Texels, targets,
 * depths and the layer rules are the serving section's.  Refused, each with a message naming its reason: plain 2-D textures and single
 * cube maps (the message names the call that serves them), 2-D arrays of section-9 formats (itw_dds_open), every format reason of
 * sections 13-16 (WIC, R32G32B32_FLOAT, UINT / SINT, R3G3B2, ...), 'DX10' dimensions other than 2, 3 and 4, array size 0, a 'DX10'
 * volume without the volume flag or with an array size above 1, a 1-D header with DDS_HEIGHT and a height other than 1, depth 0, more
 * levels than the shape allows, an item total above 2^32 - 1, width, height or depth above 16777216, and truncated payloads.
 * ------------------------------------------------------------------------------------------- */
enum { ITW_STACK_BC = 9, ITW_STACK_RAW = 13, ITW_STACK_CONVERTED = 14, ITW_STACK_OTHER_BC = 15, ITW_STACK_EXPANDED = 16 };
typedef struct itw_dds_stack_info {
    itw_dds_desc desc;        /* width, height (1 for 1-D), mip_levels, array_size (the 'DX10' count, x6 for cube maps; 1 for a
                                 volume), dxgi_format = the loaded format, is_cubemap                                             */
    uint32_t dimension;       /* 1, 2 or 3 (TEX_DIMENSION_TEXTURE1D / 2D / 3D)                                                    */
    uint32_t slices;          /* depth of level 0 of a volume, else 1                                                            */
    int32_t section;          /* ITW_STACK_*: whose decoder / converter / expansion reads the texels                             */
    int32_t form;             /* that section's header form (ITW_RAW_*, ITW_CONV_*, ITW_OBC_*, ITW_EXP_*; 0 for ITW_STACK_BC)     */
    uint64_t payload_offset;  /* where the payload starts: 128, 148 behind a 'DX10' header, or 1152 behind a palette             */
    int32_t has_alpha;        /* loadInfo.hasAlpha over every image, with the serving section's exclusions.  Taken before the cube
                                 override                                                                                        */
    int32_t has_mips, ask_user;   /* as in itw_dds_open_info                                                                     */
    /* filled by itw_dds_stack_layout, with the meanings of itw_dds_open_info: */
    int32_t layers, calls, planes;
    int32_t depth;            /* the serving section's: 8, 16 or 32 bits per channel                                             */
    int32_t width, height;    /* the top level (height 1 for a 1-D texture)                                                      */
    int32_t target_dxgi;      /* the serving section's target                                                                    */
} itw_dds_stack_info;
/* Header + the alpha check on the GPU: the serving section's scan over every image (open_alpha_kernel over an image table of every
 * item, level and slice; the byte-stream scans over the whole payload).  itw_last_kernel_ms gives the scan's time (-1 when the format
 * needs no scan).  Every refusal happens before any CUDA call.  Returns 0 on success; on failure `info` is untouched. */
int itw_dds_open_stack(const uint8_t* file, size_t size, itw_dds_stack_info* info);
/* The layout for the dialog's answers `options` (ITW_OPEN_*); pure arithmetic, no CUDA call.  Returns 0 on success. */
int itw_dds_stack_layout(itw_dds_stack_info* info, uint32_t options);
/* One DoReadContinue: the image the call reads (item `call` of a six-item texture, else slice 0 of level `call` or of level 0 / mip
 * `call` or 0 of item 0), decoded, converted or expanded by the serving section and stored into the zeroed layer, with the rules of
 * itw_dds_read_uncompressed_layer (alpha forcing of six-item textures, 16-bit planes unscaled, host or device operands, every argument
 * checked before anything is enqueued).  Only that image crosses the bus.  Returns 0 on success. */
int itw_dds_read_stack_layer(const uint8_t* file, size_t size, const itw_dds_stack_info* info, int call, void* dst, int64_t row_bytes);

/* ---------------------------------------------------------------------------------------------
 * Section 18 -- the preview dialog for HDR documents: a 32-bit document saved as BC6H_UF16, the plug-in's only HDR encoding (an
 * environment cube map, typically).  The dialog shows IDC_EXPOSURE_SLIDER for documents deeper than 16 bits (PreviewDialog.cpp:
 * 622-635): range -1000..1000, starting at 0, and each move sets exposure = float(pow(2, pos * 0.01)) and repaints both panes
 * (:868-887).  FetchPreviewRGB multiplies every float texel it shows by it (IntelPlugin.cpp:501, :649-651).  The original pane of
 * BC6H_UF16 for the cube types and for mip maps from layers is GetUncompressedImageForPreview's R16G16B16A16_FLOAT scratch converted
 * to R8G8B8A8_UNORM (:93-119, :1142-1164, :1474-1479).  DirectXTex does not hand that conversion to WIC (g_WICFormats marks the half
 * format linear and R8G8B8A8_UNORM sRGB, so _UseWICConversion returns false), so the non-WIC _Convert runs: per channel, half ->
 * float, saturate, UNORM8 store; alpha is converted too.  The rules of sections 11-17 hold: every argument is checked before
 * anything is enqueued and outputs stay untouched on failure, host and device operands are accepted (device operands: the ordering
 * rule of CompressBlocks*), the calls are synchronous, and itw_last_kernel_ms gives the time of the call's kernels.
 * Finding, reproduced and not fixed: the original pane is clamped RGBA8, so the slider brightens the compressed pane (an
 * R32G32B32A32_FLOAT display) but not the original pane; and the alpha shown in the blue slot of a mixed view moves with the slider.
 * ------------------------------------------------------------------------------------------- */
/* itw_preview_view with the dialog's exposure: FetchPreviewRGB as it runs after the slider has moved.  At depth 32 (the document or
 * an R32G32B32A32_FLOAT pane) each shown channel is FloatToByte((double)(f * exposure)), where the product is a FLOAT product,
 * rounded once and then widened.  The pure-alpha view of a source with more than 3 planes resets the exposure to 1 (:615-621); in a
 * mixture that shows alpha in the blue slot, alpha is multiplied too.  Depths 8 and 16 ignore the exposure, as the plug-in does (the
 * slider is shown at depth 32 only).  With exposure 1.0f the output equals itw_preview_view byte for byte.  Refusals: those of
 * itw_preview_view, and an exposure that is not positive and finite.  Returns 0 on success. */
int itw_preview_view_exposed(const itw_pixel_source* source, const itw_view* view, float exposure, uint8_t* dst);
/* GetUncompressedImageForPreview for encoding 95 (BC6H_UF16), in the plug-in's order:
 *   CopyDataForEncoding(DoMipMaps = false, gammaCorrect = false) through the BC6H front end (ConvertToBC6From{8,16,32}Bit) into an
 *       R16G16B16A16_FLOAT scratch
 *   cube types: the faces as itw_preview_cube builds them for 95, the chain to L when set, and the zeroed RGBA16F horizontal cross of
 *       level L (4 wL x 3 hL).  A cross without L is the converted document
 *   ITW_PANE_2D: layer 0 over the converted document (CopyLayersIntoMipMaps(..., 0, 1)) with the RGBA16F rules of
 *       itw_dds_encode_layers
 *   Convert(R16G16B16A16_FLOAT -> R8G8B8A8_UNORM, TEX_FILTER_DEFAULT): the non-WIC _Convert above, into `display`
 * `o`, `document`, `layers` and `display` as for itw_preview_uncompressed; a device display that is 4-byte aligned (pointer and
 * stride) is written in place.  `flags`: ITW_FRONT_HAS_ALPHA only.  There is no compressed size: for 95 the dialog takes it from the
 * compressed pane (itw_preview_pixels / itw_preview_cube).  Refused (besides what itw_preview_uncompressed checks): any dxgi_format
 * but 95 (itw_preview_uncompressed serves them), flips (BC6H has no normal-map column, :44-62), ITW_FRONT_GAMMA and
 * ITW_FRONT_NORMALIZE, and ITW_PANE_2D without layer 0: the plug-in builds no such pane (the dialog shows the document itself, and
 * the compressed pane comes from itw_preview_pixels).  Returns 0 on success. */
int itw_preview_uncompressed_hdr(const itw_pane_options* o, const itw_pixel_source* document, const itw_layer_source* layers,
                                 uint32_t flags, const rgba_surface* display);

#ifdef __cplusplus
}
#endif

#endif /* ITW_BCN_H */
