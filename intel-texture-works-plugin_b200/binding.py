"""ctypes binding of include/itw_bcn.h (same names, argument meaning and error behaviour)."""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def library_path():
    # ITW_BCN_LIB selects another build of the same sources (tools/tune_unroll.sh); there is no other implementation to fall back to
    return os.environ.get("ITW_BCN_LIB", os.path.join(HERE, "libitw_bcn.so"))


class RgbaSurface(ctypes.Structure):          # ispc_texcomp.h:19-25
    _fields_ = [("ptr", ctypes.c_void_p), ("width", ctypes.c_int32), ("height", ctypes.c_int32),
                ("stride", ctypes.c_int32)]


class Bc7Settings(ctypes.Structure):          # ispc_texcomp.h:27-41
    _fields_ = [("mode_selection", ctypes.c_bool * 4), ("refineIterations", ctypes.c_int * 8),
                ("skip_mode2", ctypes.c_bool), ("fastSkipTreshold_mode1", ctypes.c_int),
                ("fastSkipTreshold_mode3", ctypes.c_int), ("fastSkipTreshold_mode7", ctypes.c_int),
                ("mode45_channel0", ctypes.c_int), ("refineIterations_channel", ctypes.c_int),
                ("channels", ctypes.c_int)]


class Bc6hSettings(ctypes.Structure):         # ispc_texcomp.h:43-50
    _fields_ = [("slow_mode", ctypes.c_bool), ("fast_mode", ctypes.c_bool),
                ("refineIterations_1p", ctypes.c_int), ("refineIterations_2p", ctypes.c_int),
                ("fastSkipTreshold", ctypes.c_int)]


BC7_PROFILES = ("ultrafast", "veryfast", "fast", "basic", "slow",
                "alpha_ultrafast", "alpha_veryfast", "alpha_fast", "alpha_basic", "alpha_slow")
BC6H_PROFILES = ("bc6h_veryfast", "bc6h_fast", "bc6h_basic", "bc6h_slow", "bc6h_veryslow")

# name -> (DXGI format id, bytes per block, bytes per texel, settings kind)
FORMATS = {
    "BC1": (71, 8, 4, None), "BC3": (77, 16, 4, None), "BC4": (80, 8, 4, None), "BC5": (83, 16, 4, None),
    "BC6H": (95, 16, 8, "bc6h"), "BC7": (98, 16, 4, "bc7"),
}

EXPORTS = (["CompressBlocksBC1", "CompressBlocksBC3", "CompressBlocksBC4", "CompressBlocksBC5",
            "CompressBlocksBC6H", "CompressBlocksBC7", "itw_bytes_per_block", "itw_encode_device",
            "itw_encode_batch", "itw_set_device", "itw_get_last_error", "itw_kernel_launch_count",
            "itw_last_kernel_ms", "itw_dds_header_bytes", "itw_dds_image_bytes", "itw_dds_image_offset",
            "itw_dds_file_bytes", "itw_dds_write_header", "itw_dds_read_header", "itw_dds_encode_file",
            "itw_mip_scratch_bytes", "itw_generate_mips_device", "itw_dds_encode_texture", "itw_decode", "itw_convert_pixels", "itw_encode_pixels",
            "itw_generate_mips_device_f16", "itw_generate_mips_device_srgb", "itw_dds_encode_pixels", "itw_release", "itw_set_devices", "itw_get_devices",
            "itw_begin_deferred", "itw_flush", "GetProcessorCount", "InitWin32Threads", "DestroyThreads", "GetBytesPerBlock",
            "CompressImageMT", "CompressImageST", "CompressImageBC1", "CompressImageBC3",
            "itw_shard_plan_make", "itw_shard_unique_id", "itw_shard_init", "itw_shard_finalize", "itw_encode_mip_chain_sharded",
            "itw_decompress", "itw_preview_pixels", "itw_dds_open", "itw_dds_open_layout", "itw_dds_read_layer",
            "itw_dds_encode_layers", "itw_cube_layout", "itw_dds_encode_cube", "itw_preview_cube", "itw_preview_layers", "itw_preview_view",
            "itw_preview_uncompressed", "itw_dds_none_layout", "itw_dds_save_none", "itw_dds_open_uncompressed", "itw_dds_uncompressed_layout",
            "itw_dds_read_uncompressed_layer", "itw_dds_open_converted", "itw_dds_converted_layout", "itw_dds_read_converted_layer",
            "itw_dds_open_other_bc", "itw_dds_other_bc_layout", "itw_dds_read_other_bc_layer", "itw_dds_open_expanded",
            "itw_dds_expanded_layout", "itw_dds_read_expanded_layer", "itw_dds_open_stack", "itw_dds_stack_layout",
            "itw_dds_read_stack_layer", "itw_preview_view_exposed", "itw_preview_uncompressed_hdr"]
           + ["CompressImageBC7_" + p for p in BC7_PROFILES] + ["CompressImage" + p.replace("bc6h_", "BC6H_") for p in BC6H_PROFILES]
           + ["GetProfile_" + p for p in BC7_PROFILES + BC6H_PROFILES])


class PixelSource(ctypes.Structure):          # include/itw_bcn.h section 6
    _fields_ = [("data", ctypes.c_void_p), ("width", ctypes.c_int32), ("height", ctypes.c_int32), ("planes", ctypes.c_int32),
                ("depth", ctypes.c_int32), ("row_bytes", ctypes.c_int64)]


class LayerSource(ctypes.Structure):          # include/itw_bcn.h section 6
    _fields_ = [("channels", ctypes.c_void_p * 3), ("channel_count", ctypes.c_int32), ("alpha", ctypes.c_void_p),
                ("row_bytes", ctypes.c_int64)]


FRONT_HAS_ALPHA, FRONT_GAMMA, FRONT_FLIP_X, FRONT_FLIP_Y, FRONT_NORMALIZE = 1, 2, 4, 8, 16


class DdsDesc(ctypes.Structure):              # include/itw_bcn.h section 3
    _fields_ = [("width", ctypes.c_uint32), ("height", ctypes.c_uint32), ("mip_levels", ctypes.c_uint32),
                ("array_size", ctypes.c_uint32), ("dxgi_format", ctypes.c_uint32), ("is_cubemap", ctypes.c_uint32)]


class DdsOpenInfo(ctypes.Structure):         # include/itw_bcn.h section 9
    _fields_ = [("desc", DdsDesc), ("has_alpha", ctypes.c_int32), ("has_mips", ctypes.c_int32), ("ask_user", ctypes.c_int32),
                ("layers", ctypes.c_int32), ("calls", ctypes.c_int32), ("planes", ctypes.c_int32), ("depth", ctypes.c_int32),
                ("width", ctypes.c_int32), ("height", ctypes.c_int32), ("target_dxgi", ctypes.c_int32)]


OPEN_SEPARATE_ALPHA, OPEN_MIPS = 1, 2


class DdsUncompressedInfo(ctypes.Structure):  # include/itw_bcn.h section 13
    _fields_ = [("desc", DdsDesc), ("source", ctypes.c_int32), ("payload_offset", ctypes.c_uint64), ("has_alpha", ctypes.c_int32),
                ("has_mips", ctypes.c_int32), ("ask_user", ctypes.c_int32), ("layers", ctypes.c_int32), ("calls", ctypes.c_int32),
                ("planes", ctypes.c_int32), ("depth", ctypes.c_int32), ("width", ctypes.c_int32), ("height", ctypes.c_int32),
                ("target_dxgi", ctypes.c_int32)]


RAW_DX10, RAW_A8B8G8R8, RAW_X8B8G8R8, RAW_R8G8B8, RAW_A16B16G16R16, RAW_A32B32G32R32F = 0, 1, 2, 3, 4, 5


class DdsConvertedInfo(ctypes.Structure):     # include/itw_bcn.h section 14
    _fields_ = [("desc", DdsDesc), ("form", ctypes.c_int32), ("payload_offset", ctypes.c_uint64), ("has_alpha", ctypes.c_int32),
                ("has_mips", ctypes.c_int32), ("ask_user", ctypes.c_int32), ("layers", ctypes.c_int32), ("calls", ctypes.c_int32),
                ("planes", ctypes.c_int32), ("depth", ctypes.c_int32), ("width", ctypes.c_int32), ("height", ctypes.c_int32),
                ("target_dxgi", ctypes.c_int32)]


(CONV_DX10, CONV_G16R16, CONV_A8L8, CONV_A8, CONV_A4R4G4B4, CONV_X4R4G4B4, CONV_Q16W16V16U16, CONV_R16F, CONV_G16R16F,
 CONV_A16B16G16R16F, CONV_G32R32F) = range(11)


class DdsOtherBcInfo(ctypes.Structure):       # include/itw_bcn.h section 15: the fields of section 14
    _fields_ = DdsConvertedInfo._fields_


OBC_DX10, OBC_DXT3, OBC_DXT2, OBC_DXT4, OBC_BC4S, OBC_BC5S = range(6)


class DdsExpandedInfo(ctypes.Structure):      # include/itw_bcn.h section 16: the fields of section 14
    _fields_ = DdsConvertedInfo._fields_


EXP_P8, EXP_A8P8, EXP_A8R3G3B2, EXP_A4L4 = range(4)


class DdsStackInfo(ctypes.Structure):         # include/itw_bcn.h section 17
    _fields_ = [("desc", DdsDesc), ("dimension", ctypes.c_uint32), ("slices", ctypes.c_uint32), ("section", ctypes.c_int32),
                ("form", ctypes.c_int32)] + DdsConvertedInfo._fields_[2:]


STACK_BC, STACK_RAW, STACK_CONVERTED, STACK_OTHER_BC, STACK_EXPANDED = 9, 13, 14, 15, 16


class CubeOptions(ctypes.Structure):          # include/itw_bcn.h section 10
    _fields_ = [("dxgi_format", ctypes.c_uint32), ("source", ctypes.c_int32), ("mip_maps", ctypes.c_int32), ("mip_level", ctypes.c_int32)]


CUBE_CROSS, CUBE_LAYERS = 0, 1


class View(ctypes.Structure):                 # include/itw_bcn.h section 11
    _fields_ = [("width", ctypes.c_int32), ("height", ctypes.c_int32), ("x", ctypes.c_int32), ("y", ctypes.c_int32),
                ("zoom", ctypes.c_double), ("mip_level", ctypes.c_int32), ("channels", ctypes.c_uint32), ("matte", ctypes.c_uint32)]


VIEW_RED, VIEW_GREEN, VIEW_BLUE, VIEW_ALPHA = 0x4, 0x8, 0x10, 0x20


class PaneOptions(ctypes.Structure):          # include/itw_bcn.h section 11
    _fields_ = [("dxgi_format", ctypes.c_uint32), ("texture", ctypes.c_int32), ("mip_level", ctypes.c_int32)]


PANE_2D, PANE_CUBE_CROSS, PANE_CUBE_LAYERS = 0, 1, 2


class NoneOptions(ctypes.Structure):          # include/itw_bcn.h section 12
    _fields_ = [("texture", ctypes.c_int32), ("mip_maps", ctypes.c_int32), ("mip_level", ctypes.c_int32)]


class ShardPlan(ctypes.Structure):            # include/itw_bcn.h section 7
    _fields_ = [("nranks", ctypes.c_int32), ("rank", ctypes.c_int32), ("levels", ctypes.c_int32), ("band_levels", ctypes.c_int32),
                ("band_y0", ctypes.c_int32), ("band_y1", ctypes.c_int32), ("slot_bytes", ctypes.c_uint64), ("chain_bytes", ctypes.c_uint64),
                ("level_offset", ctypes.c_uint64 * 16), ("level_bytes", ctypes.c_uint64 * 16), ("send_offset", ctypes.c_uint64 * 16),
                ("band_bytes", ctypes.c_uint64 * 16), ("texel_offset", ctypes.c_uint64), ("texel_bytes", ctypes.c_uint64)]


class EncoderApi:
    """A loaded library exporting the reference C-ABI (optionally with a symbol prefix).

    Used for the product (prefix "") and, by tests only, for the oracle ("oracle_"), the
    reference-source build ("") and the CPU emulation ("emu_")."""

    def __init__(self, path, prefix=""):
        if not os.path.exists(path):
            raise FileNotFoundError(f"{path} is missing -- build it first (python __graft_entry__.py build)")
        self.path = path
        self.prefix = prefix
        self.lib = ctypes.CDLL(path)

    def fn(self, name):
        return getattr(self.lib, self.prefix + name)

    def profile(self, name):
        """Settings struct filled by GetProfile_<name> (zero-initialised first, like the canonical model)."""
        s = Bc6hSettings() if name.startswith("bc6h_") else Bc7Settings()
        f = self.fn("GetProfile_" + name)
        f.restype = None
        f(ctypes.byref(s))
        return s

    def _call(self, fmt, surf, dst_ptr, settings):
        f = self.fn("CompressBlocks" + fmt)
        f.restype = None
        kind = FORMATS[fmt][3]
        if kind is None:
            f(ctypes.byref(surf), ctypes.c_void_p(dst_ptr))
        else:
            if settings is None:
                raise ValueError(f"{fmt} needs a settings struct")
            f(ctypes.byref(surf), ctypes.c_void_p(dst_ptr), ctypes.byref(settings))

    def encode(self, fmt, image, settings=None):
        """Encode a host numpy image (H x W x 4, uint8 for LDR / uint16 half bits for BC6H)."""
        _, bpb, texel, _ = FORMATS[fmt]
        h, w = image.shape[:2]
        assert image.strides[1] == texel and image.shape[2] * image.itemsize == texel, "RGBA8 / RGBA16F texels expected"
        surf = RgbaSurface(image.ctypes.data, w, h, image.strides[0])
        out = np.zeros((h // 4) * (w // 4) * bpb, dtype=np.uint8)
        self._call(fmt, surf, out.ctypes.data, settings)
        self.check()
        return out

    def decode(self, fmt, blocks, width, height):
        """itw_decode: host blocks -> H x W x 4 image (uint8; uint16 half bit patterns for BC6H)."""
        _, bpb, texel, _ = FORMATS[fmt]
        blocks = np.ascontiguousarray(np.frombuffer(bytes(blocks), np.uint8))
        assert blocks.size == (width // 4) * (height // 4) * bpb
        img = np.zeros((height, width, 4), np.uint16 if texel == 8 else np.uint8)
        self.decode_raw(fmt, blocks.ctypes.data, img.ctypes.data, width, height, img.strides[0])
        return img

    def decode_raw(self, fmt, blocks_ptr, dst_ptr, width, height, stride):
        """itw_decode on raw addresses (host or device)."""
        f = self.fn("itw_decode")
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(RgbaSurface)]
        surf = RgbaSurface(dst_ptr, width, height, stride)
        rc = f(FORMATS[fmt][0], ctypes.c_void_p(blocks_ptr), ctypes.byref(surf))
        self.check()
        if rc != 0:
            raise RuntimeError("itw_decode failed")

    def convert_pixels(self, fmt, pixels, flags=0, pad=True):
        """itw_convert_pixels: host numpy H x W x planes array (uint8 / uint16 / float32) -> RGBA8 / RGBA16F image."""
        h, w, planes = pixels.shape
        pixels = np.ascontiguousarray(pixels)
        texel = FORMATS[fmt][2]
        dw, dh = ((w + 3) & ~3, (h + 3) & ~3) if pad else (w, h)
        img = np.zeros((dh, dw, 4), np.uint16 if texel == 8 else np.uint8)
        src = PixelSource(pixels.ctypes.data, w, h, planes, pixels.itemsize * 8, 0)
        self.convert_pixels_raw(fmt, src, flags, img.ctypes.data, dw, dh, img.strides[0])
        return img

    def convert_pixels_raw(self, fmt, src, flags, dst_ptr, width, height, stride):
        f = self.fn("itw_convert_pixels")
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_int, ctypes.POINTER(PixelSource), ctypes.c_uint32, ctypes.POINTER(RgbaSurface)]
        surf = RgbaSurface(dst_ptr, width, height, stride)
        rc = f(FORMATS[fmt][0], ctypes.byref(src), flags, ctypes.byref(surf))
        self.check()
        if rc != 0:
            raise RuntimeError("itw_convert_pixels failed")

    def encode_raw(self, fmt, ptr, width, height, stride, dst_ptr, settings=None):
        """CompressBlocks<fmt> on raw addresses (host or device)."""
        self._call(fmt, RgbaSurface(ptr, width, height, stride), dst_ptr, settings)
        self.check()

    def check(self):
        pass


class ItwBcn(EncoderApi):
    """The product library.  Raises on any reported error; never falls back to a CPU path."""

    def __init__(self, path=None):
        super().__init__(path or library_path())
        L = self.lib
        L.itw_get_last_error.restype = ctypes.c_char_p
        L.itw_kernel_launch_count.restype = ctypes.c_uint64
        L.itw_last_kernel_ms.restype = ctypes.c_float
        L.itw_encode_device.restype = ctypes.c_int
        L.itw_encode_device.argtypes = [ctypes.c_int, ctypes.POINTER(RgbaSurface), ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_void_p]
        L.itw_encode_batch.restype = ctypes.c_int
        L.itw_bytes_per_block.restype = ctypes.c_int
        L.itw_set_device.restype = ctypes.c_int

        for n in ("itw_dds_header_bytes", "itw_dds_image_bytes", "itw_dds_image_offset", "itw_dds_file_bytes",
                  "itw_dds_write_header", "itw_dds_read_header", "itw_dds_encode_file"):
            getattr(L, n).restype = ctypes.c_size_t
        L.itw_dds_image_bytes.argtypes = [ctypes.POINTER(DdsDesc), ctypes.c_uint32]
        L.itw_dds_image_offset.argtypes = [ctypes.POINTER(DdsDesc), ctypes.c_uint32, ctypes.c_uint32]
        L.itw_dds_write_header.argtypes = [ctypes.POINTER(DdsDesc), ctypes.c_void_p, ctypes.c_size_t]
        L.itw_dds_read_header.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsDesc)]
        L.itw_dds_encode_file.argtypes = [ctypes.POINTER(DdsDesc), ctypes.POINTER(RgbaSurface), ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_size_t]

        L.itw_mip_scratch_bytes.restype = ctypes.c_size_t
        L.itw_generate_mips_device.restype = ctypes.c_int
        L.itw_generate_mips_device.argtypes = [ctypes.POINTER(RgbaSurface), ctypes.c_int, ctypes.POINTER(RgbaSurface),
                                               ctypes.c_void_p, ctypes.c_void_p]
        L.itw_dds_encode_texture.restype = ctypes.c_size_t
        L.itw_dds_encode_texture.argtypes = [ctypes.POINTER(DdsDesc), ctypes.POINTER(RgbaSurface), ctypes.c_void_p,
                                             ctypes.c_void_p, ctypes.c_size_t]

    def encode_pixels(self, fmt, pixels, flags=0, settings=None):
        """itw_encode_pixels: host numpy H x W x planes array -> blocks of the padded image."""
        h, w, planes = pixels.shape
        pixels = np.ascontiguousarray(pixels)
        out = np.zeros(((w + 3) // 4) * ((h + 3) // 4) * FORMATS[fmt][1], np.uint8)
        src = PixelSource(pixels.ctypes.data, w, h, planes, pixels.itemsize * 8, 0)
        self.encode_pixels_raw(fmt, src, flags, out.ctypes.data, settings)
        return out

    def encode_pixels_raw(self, fmt, src, flags, dst_ptr, settings=None):
        f = self.lib.itw_encode_pixels
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_int, ctypes.POINTER(PixelSource), ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        rc = f(FORMATS[fmt][0], ctypes.byref(src), flags, sp, ctypes.c_void_p(dst_ptr))
        self.check()
        if rc != 0:
            raise RuntimeError("itw_encode_pixels failed")

    def last_error(self):
        return self.lib.itw_get_last_error().decode()

    def dds_encode_texture(self, desc, tops, settings=None):
        """itw_dds_encode_texture: `tops` = host numpy level-0 images (one per array item); mips made on the GPU."""
        n = self.lib.itw_dds_file_bytes(ctypes.byref(desc))
        if not n:
            raise ValueError("unsupported DDS description")
        surf = (RgbaSurface * len(tops))(*[RgbaSurface(im.ctypes.data, im.shape[1], im.shape[0], im.strides[0]) for im in tops])
        out = np.zeros(n, np.uint8)
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        got = self.lib.itw_dds_encode_texture(ctypes.byref(desc), surf, sp, out.ctypes.data, n)
        if got != n:
            self.check()
            raise RuntimeError("itw_dds_encode_texture failed")
        return out

    def dds_encode_pixels(self, desc, pixel_arrays, flags=0, settings=None):
        """itw_dds_encode_pixels: `pixel_arrays` = host numpy H x W x planes arrays (one per array item); the plug-in's whole save path."""
        n = self.lib.itw_dds_file_bytes(ctypes.byref(desc))
        if not n:
            raise ValueError("unsupported DDS description")
        keep = [np.ascontiguousarray(a) for a in pixel_arrays]
        srcs = (PixelSource * len(keep))(*[PixelSource(a.ctypes.data, a.shape[1], a.shape[0], a.shape[2], a.itemsize * 8, 0) for a in keep])
        out = np.zeros(n, np.uint8)
        f = self.lib.itw_dds_encode_pixels
        f.restype = ctypes.c_size_t
        f.argtypes = [ctypes.POINTER(DdsDesc), ctypes.POINTER(PixelSource), ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        got = f(ctypes.byref(desc), srcs, flags, sp, out.ctypes.data, n)
        if got != n:
            self.check()
            raise RuntimeError("itw_dds_encode_pixels failed")
        return out

    def dds_encode_layers(self, desc, composite, layers, flags=0, settings=None):
        """itw_dds_encode_layers: `composite` = host numpy H x W x planes array; `layers` = one entry per document layer, each a
        (channels, alpha) pair: 1..3 H x W numpy planes of the composite's dtype, and an H x W plane or None (white)."""
        n = self.lib.itw_dds_file_bytes(ctypes.byref(desc))
        if not n:
            raise ValueError("unsupported DDS description")
        comp = np.ascontiguousarray(composite)
        keep = []
        srcs = (LayerSource * max(1, len(layers)))()
        for i, (channels, alpha) in enumerate(layers):
            planes = [np.ascontiguousarray(c, comp.dtype) for c in channels]
            a = None if alpha is None else np.ascontiguousarray(alpha, comp.dtype)
            keep += planes + [a]
            srcs[i].channel_count = len(planes)
            for c, pl in enumerate(planes):
                srcs[i].channels[c] = pl.ctypes.data
            srcs[i].alpha = None if a is None else a.ctypes.data
            srcs[i].row_bytes = 0
        src = PixelSource(comp.ctypes.data, comp.shape[1], comp.shape[0], comp.shape[2], comp.itemsize * 8, 0)
        out = np.zeros(n, np.uint8)
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        got = self.dds_encode_layers_raw(desc, src, srcs, len(layers), flags, sp, out.ctypes.data, n)
        if got != n:
            self.check()
            raise RuntimeError("itw_dds_encode_layers failed: " + self.last_error())
        return out

    def dds_encode_layers_raw(self, desc, composite, layers, count, flags, settings_ptr, file_ptr, capacity):
        """itw_dds_encode_layers on ctypes structures and raw addresses; returns the file size (0 on error)."""
        f = self.lib.itw_dds_encode_layers
        f.restype = ctypes.c_size_t
        f.argtypes = [ctypes.POINTER(DdsDesc), ctypes.POINTER(PixelSource), ctypes.POINTER(LayerSource), ctypes.c_int, ctypes.c_uint32,
                      ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t]
        return f(ctypes.byref(desc), ctypes.byref(composite), layers, count, flags, settings_ptr, file_ptr, capacity)

    def dds_encode_file(self, desc, images, settings=None):
        """itw_dds_encode_file: `images` = host numpy arrays, item-major / mip-minor, padded to multiples of 4."""
        n = self.lib.itw_dds_file_bytes(ctypes.byref(desc))
        if not n:
            raise ValueError("unsupported DDS description")
        surf = (RgbaSurface * len(images))(*[RgbaSurface(im.ctypes.data, im.shape[1], im.shape[0], im.strides[0]) for im in images])
        out = np.zeros(n, np.uint8)
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        got = self.lib.itw_dds_encode_file(ctypes.byref(desc), surf, sp, out.ctypes.data, n)
        if got != n:
            self.check()
            raise RuntimeError("itw_dds_encode_file failed")
        return out

    def cube_layout(self, options, doc_width, doc_height):
        """itw_cube_layout: (file size, DdsDesc, face width, face height); size 0 (and the error text) when refused."""
        f = self.lib.itw_cube_layout
        f.restype = ctypes.c_size_t
        f.argtypes = [ctypes.POINTER(CubeOptions), ctypes.c_int, ctypes.c_int, ctypes.POINTER(DdsDesc), ctypes.POINTER(ctypes.c_int),
                      ctypes.POINTER(ctypes.c_int)]
        d, fw, fh = DdsDesc(), ctypes.c_int(0), ctypes.c_int(0)
        n = f(ctypes.byref(options), doc_width, doc_height, ctypes.byref(d), ctypes.byref(fw), ctypes.byref(fh))
        return n, d, fw.value, fh.value

    @staticmethod
    def cube_faces(faces, dtype, keep):
        """Six LayerSource from `faces`: per face None (no layer of that name) or (channels, alpha) as dds_encode_layers takes them."""
        arr = (LayerSource * 6)()
        for i, face in enumerate(faces):
            if face is None:
                continue
            channels, alpha = face
            planes = [np.ascontiguousarray(c, dtype) for c in channels]
            a = None if alpha is None else np.ascontiguousarray(alpha, dtype)
            keep += planes + [a]
            arr[i].channel_count = len(planes)
            for c, pl in enumerate(planes):
                arr[i].channels[c] = pl.ctypes.data
            arr[i].alpha = None if a is None else a.ctypes.data
        return arr

    def dds_encode_cube(self, options, document, faces=None, flags=0, settings=None):
        """itw_dds_encode_cube: `document` = host numpy H x W x planes array (the cross, or the composite that gives the size and depth
        of a layer cube); `faces` = six entries as cube_faces takes them (layer cubes only)."""
        doc = np.ascontiguousarray(document)
        n = self.cube_layout(options, doc.shape[1], doc.shape[0])[0]
        if not n:
            raise ValueError("itw_cube_layout refused the options: " + self.last_error())
        keep = []
        arr = self.cube_faces(faces, doc.dtype, keep) if faces is not None else None
        src = PixelSource(doc.ctypes.data, doc.shape[1], doc.shape[0], doc.shape[2], doc.itemsize * 8, 0)
        out = np.zeros(n, np.uint8)
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        got = self.dds_encode_cube_raw(options, src, arr, flags, sp, out.ctypes.data, n)
        if got != n:
            raise RuntimeError("itw_dds_encode_cube failed: " + self.last_error())
        return out

    def dds_encode_cube_raw(self, options, document, faces, flags, settings_ptr, file_ptr, capacity):
        """itw_dds_encode_cube on ctypes structures and raw addresses; returns the file size (0 on error)."""
        f = self.lib.itw_dds_encode_cube
        f.restype = ctypes.c_size_t
        f.argtypes = [ctypes.POINTER(CubeOptions), ctypes.POINTER(PixelSource), ctypes.POINTER(LayerSource), ctypes.c_uint32, ctypes.c_void_p,
                      ctypes.c_void_p, ctypes.c_size_t]
        return f(ctypes.byref(options), ctypes.byref(document), faces, flags, settings_ptr, file_ptr, capacity)

    def preview_cube(self, options, document, faces=None, flags=0, settings=None):
        """itw_preview_cube on host arrays (as dds_encode_cube) -> (display image, compressed bytes).  The display is the document
        (a cross without a set level) or the 4 wL x 3 hL cross; float32 for BC6H at depth 32, uint8 otherwise."""
        doc = np.ascontiguousarray(document)
        n, d, fw, fh = self.cube_layout(options, doc.shape[1], doc.shape[0])
        if not n:
            raise ValueError("itw_cube_layout refused the options: " + self.last_error())
        if options.source == CUBE_CROSS and options.mip_level < 0:
            w, h = doc.shape[1], doc.shape[0]
        else:
            w, h = 4 * d.width, 3 * d.height
        img = np.zeros((h, w, 4), np.float32 if (options.dxgi_format == 95 and doc.itemsize == 4) else np.uint8)
        keep = []
        arr = self.cube_faces(faces, doc.dtype, keep) if faces is not None else None
        src = PixelSource(doc.ctypes.data, doc.shape[1], doc.shape[0], doc.shape[2], doc.itemsize * 8, 0)
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        size = ctypes.c_size_t(0)
        rc = self.preview_cube_raw(options, src, arr, flags, sp, RgbaSurface(img.ctypes.data, w, h, img.strides[0]), ctypes.byref(size))
        if rc != 0:
            raise RuntimeError("itw_preview_cube failed: " + self.last_error())
        return img, size.value

    def preview_cube_raw(self, options, document, faces, flags, settings_ptr, display, size_ref):
        """itw_preview_cube on ctypes structures; returns its status."""
        f = self.lib.itw_preview_cube
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(CubeOptions), ctypes.POINTER(PixelSource), ctypes.POINTER(LayerSource), ctypes.c_uint32, ctypes.c_void_p,
                      ctypes.POINTER(RgbaSurface), ctypes.POINTER(ctypes.c_size_t)]
        return f(ctypes.byref(options), ctypes.byref(document), faces, flags, settings_ptr, ctypes.byref(display), size_ref)

    def decompress(self, dxgi_format, blocks, width, height, target):
        """itw_decompress: host blocks -> H x W x 4 image of `target` (uint8 for 28 / 29, float32 for 2)."""
        blocks = np.ascontiguousarray(np.frombuffer(bytes(blocks), np.uint8))
        img = np.zeros((height, width, 4), np.float32 if target == 2 else np.uint8)
        self.decompress_raw(dxgi_format, blocks.ctypes.data, width, height, target, img.ctypes.data, img.strides[0])
        return img

    def decompress_raw(self, dxgi_format, blocks_ptr, width, height, target, dst_ptr, stride):
        """itw_decompress on raw addresses (host or device)."""
        f = self.lib.itw_decompress
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(RgbaSurface)]
        rc = f(dxgi_format, ctypes.c_void_p(blocks_ptr), width, height, target, ctypes.byref(RgbaSurface(dst_ptr, width, height, stride)))
        self.check()
        if rc != 0:
            raise RuntimeError("itw_decompress failed")

    def preview_pixels(self, dxgi_format, faces, flags=0, settings=None):
        """itw_preview_pixels: `faces` = one or six host numpy H x W x planes arrays -> (display image, compressed bytes).  The
        display is float32 for BC6H at depth 32, uint8 otherwise; a cube map gives the 4w x 3h cross."""
        keep = [np.ascontiguousarray(a) for a in faces]
        h, w = keep[0].shape[:2]
        if len(keep) == 6:
            w, h = 4 * w, 3 * h
        hdr = dxgi_format in (95, 96) and keep[0].itemsize == 4
        img = np.zeros((h, w, 4), np.float32 if hdr else np.uint8)
        srcs = (PixelSource * len(keep))(*[PixelSource(a.ctypes.data, a.shape[1], a.shape[0], a.shape[2], a.itemsize * 8, 0) for a in keep])
        n = self.preview_pixels_raw(dxgi_format, srcs, len(keep), flags, settings, img.ctypes.data, w, h, img.strides[0])
        return img, n

    def preview_pixels_raw(self, dxgi_format, sources, count, flags, settings, dst_ptr, width, height, stride):
        f = self.lib.itw_preview_pixels
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_int, ctypes.POINTER(PixelSource), ctypes.c_int, ctypes.c_uint32, ctypes.c_void_p,
                      ctypes.POINTER(RgbaSurface), ctypes.POINTER(ctypes.c_size_t)]
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        n = ctypes.c_size_t(0)
        rc = f(dxgi_format, sources, count, flags, sp, ctypes.byref(RgbaSurface(dst_ptr, width, height, stride)), ctypes.byref(n))
        self.check()
        if rc != 0:
            raise RuntimeError("itw_preview_pixels failed")
        return n.value

    def preview_layers(self, dxgi_format, composite, layer0, flags=0, settings=None):
        """itw_preview_layers: `composite` = host numpy H x W x planes array, `layer0` = (channels, alpha) as dds_encode_layers takes
        one layer -> (display image, compressed bytes).  The display is float32 for BC6H at depth 32, uint8 otherwise."""
        comp = np.ascontiguousarray(composite)
        h, w = comp.shape[:2]
        keep = []
        arr = (LayerSource * 1)()
        channels, alpha = layer0
        planes = [np.ascontiguousarray(c, comp.dtype) for c in channels]
        a = None if alpha is None else np.ascontiguousarray(alpha, comp.dtype)
        keep += planes + [a]
        arr[0].channel_count = len(planes)
        for c, pl in enumerate(planes):
            arr[0].channels[c] = pl.ctypes.data
        arr[0].alpha = None if a is None else a.ctypes.data
        img = np.zeros((h, w, 4), np.float32 if (dxgi_format in (95, 96) and comp.itemsize == 4) else np.uint8)
        src = PixelSource(comp.ctypes.data, w, h, comp.shape[2], comp.itemsize * 8, 0)
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        size = ctypes.c_size_t(0)
        rc = self.preview_layers_raw(dxgi_format, src, arr, flags, sp, RgbaSurface(img.ctypes.data, w, h, img.strides[0]), ctypes.byref(size))
        if rc != 0:
            raise RuntimeError("itw_preview_layers failed: " + self.last_error())
        return img, size.value

    def preview_layers_raw(self, dxgi_format, composite, layer0, flags, settings_ptr, display, size_ref):
        """itw_preview_layers on ctypes structures; returns its status."""
        f = self.lib.itw_preview_layers
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_int, ctypes.POINTER(PixelSource), ctypes.POINTER(LayerSource), ctypes.c_uint32, ctypes.c_void_p,
                      ctypes.POINTER(RgbaSurface), ctypes.POINTER(ctypes.c_size_t)]
        return f(dxgi_format, ctypes.byref(composite), layer0, flags, settings_ptr, ctypes.byref(display), size_ref)

    def preview_view(self, source, view):
        """itw_preview_view: `source` = host numpy H x W x planes array (uint8 depth 8, uint16 depth 16, float32 depth 32: the
        document, or a pane of itw_preview_pixels), `view` = a View -> the view->height x view->width x 3 uint8 dialog buffer."""
        src = np.ascontiguousarray(source)
        out = np.zeros((view.height, view.width, 3), np.uint8)
        ps = PixelSource(src.ctypes.data, src.shape[1], src.shape[0], src.shape[2], src.itemsize * 8, 0)
        if self.preview_view_raw(ps, view, out.ctypes.data) != 0:
            raise RuntimeError("itw_preview_view failed: " + self.last_error())
        return out

    def preview_view_raw(self, source, view, dst_ptr):
        """itw_preview_view on ctypes structures and a raw (host or device) address; returns its status."""
        f = self.lib.itw_preview_view
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(PixelSource), ctypes.POINTER(View), ctypes.c_void_p]
        return f(ctypes.byref(source) if source is not None else None, ctypes.byref(view) if view is not None else None,
                 ctypes.c_void_p(dst_ptr) if dst_ptr else None)

    def preview_view_exposed(self, source, view, exposure):
        """itw_preview_view_exposed: preview_view with the dialog's exposure (a float; the slider's float(2 ** (pos * 0.01)))."""
        src = np.ascontiguousarray(source)
        out = np.zeros((view.height, view.width, 3), np.uint8)
        ps = PixelSource(src.ctypes.data, src.shape[1], src.shape[0], src.shape[2], src.itemsize * 8, 0)
        if self.preview_view_exposed_raw(ps, view, exposure, out.ctypes.data) != 0:
            raise RuntimeError("itw_preview_view_exposed failed: " + self.last_error())
        return out

    def preview_view_exposed_raw(self, source, view, exposure, dst_ptr):
        """itw_preview_view_exposed on ctypes structures and a raw (host or device) address; returns its status."""
        f = self.lib.itw_preview_view_exposed
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(PixelSource), ctypes.POINTER(View), ctypes.c_float, ctypes.c_void_p]
        return f(ctypes.byref(source) if source is not None else None, ctypes.byref(view) if view is not None else None, exposure,
                 ctypes.c_void_p(dst_ptr) if dst_ptr else None)

    def preview_uncompressed(self, options, document, layers=None, flags=0):
        """itw_preview_uncompressed on host arrays -> (uint8 H x W x 4 pane, compressed bytes).  `document` = host numpy H x W x planes
        array; `layers` = None, or for PANE_2D one layer (channels, alpha) and for PANE_CUBE_LAYERS six entries as cube_faces takes
        them.  The pane is the document's size (2-D, or a cross without a set level) or the 4 wL x 3 hL cross of level L."""
        doc = np.ascontiguousarray(document)
        dh, dw = doc.shape[:2]
        w, h = self.pane_size(options, dw, dh)
        keep = []
        arr = None
        if layers is not None:
            arr = self.cube_faces([layers] if options.texture == PANE_2D else layers, doc.dtype, keep)
        img = np.zeros((h, w, 4), np.uint8)
        src = PixelSource(doc.ctypes.data, dw, dh, doc.shape[2], doc.itemsize * 8, 0)
        size = ctypes.c_size_t(0)
        rc = self.preview_uncompressed_raw(options, src, arr, flags, RgbaSurface(img.ctypes.data, w, h, img.strides[0]), ctypes.byref(size))
        if rc != 0:
            raise RuntimeError("itw_preview_uncompressed failed: " + self.last_error())
        return img, size.value

    def preview_uncompressed_raw(self, options, document, layers, flags, display, size_ref):
        """itw_preview_uncompressed on ctypes structures (any of them may be None); returns its status."""
        f = self.lib.itw_preview_uncompressed
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(PaneOptions), ctypes.POINTER(PixelSource), ctypes.POINTER(LayerSource), ctypes.c_uint32,
                      ctypes.POINTER(RgbaSurface), ctypes.POINTER(ctypes.c_size_t)]
        ref = lambda x: ctypes.byref(x) if x is not None else None
        return f(ref(options), ref(document), layers, flags, ref(display), size_ref)

    def preview_uncompressed_hdr(self, options, document, layers=None, flags=0):
        """itw_preview_uncompressed_hdr on host arrays -> the uint8 H x W x 4 pane of BC6H_UF16 (options.dxgi_format 95); arguments
        and pane size as for preview_uncompressed."""
        doc = np.ascontiguousarray(document)
        w, h = self.pane_size(options, doc.shape[1], doc.shape[0])
        keep = []
        arr = None
        if layers is not None:
            arr = self.cube_faces([layers] if options.texture == PANE_2D else layers, doc.dtype, keep)
        img = np.zeros((h, w, 4), np.uint8)
        src = PixelSource(doc.ctypes.data, doc.shape[1], doc.shape[0], doc.shape[2], doc.itemsize * 8, 0)
        if self.preview_uncompressed_hdr_raw(options, src, arr, flags, RgbaSurface(img.ctypes.data, w, h, img.strides[0])) != 0:
            raise RuntimeError("itw_preview_uncompressed_hdr failed: " + self.last_error())
        return img

    def preview_uncompressed_hdr_raw(self, options, document, layers, flags, display):
        """itw_preview_uncompressed_hdr on ctypes structures (any of them may be None); returns its status."""
        f = self.lib.itw_preview_uncompressed_hdr
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(PaneOptions), ctypes.POINTER(PixelSource), ctypes.POINTER(LayerSource), ctypes.c_uint32,
                      ctypes.POINTER(RgbaSurface)]
        ref = lambda x: ctypes.byref(x) if x is not None else None
        return f(ref(options), ref(document), layers, flags, ref(display))

    @staticmethod
    def pane_size(options, dw, dh):
        """(width, height) of an uncompressed pane: the document's (2-D, or a cross without a set level), else the 4 wL x 3 hL cross."""
        if options.texture == PANE_2D or (options.texture == PANE_CUBE_CROSS and options.mip_level < 0):
            return dw, dh
        fw, fh = (dw, dh) if options.texture == PANE_CUBE_LAYERS else ((dw // 3, dh // 4) if dw < dh else (dw // 4, dh // 3))
        L = max(options.mip_level, 0)
        return 4 * max(1, fw >> L), 3 * max(1, fh >> L)

    def none_layout(self, options, doc_width, doc_height):
        """itw_dds_none_layout: (file size, DdsDesc, level-0 width, level-0 height); size 0 (and the error text) when refused."""
        f = self.lib.itw_dds_none_layout
        f.restype = ctypes.c_size_t
        f.argtypes = [ctypes.POINTER(NoneOptions), ctypes.c_int, ctypes.c_int, ctypes.POINTER(DdsDesc), ctypes.POINTER(ctypes.c_int),
                      ctypes.POINTER(ctypes.c_int)]
        d, fw, fh = DdsDesc(), ctypes.c_int(0), ctypes.c_int(0)
        n = f(ctypes.byref(options) if options is not None else None, doc_width, doc_height, ctypes.byref(d), ctypes.byref(fw), ctypes.byref(fh))
        return n, d, fw.value, fh.value

    def dds_save_none(self, options, document, layers=None, flags=0):
        """itw_dds_save_none on host arrays -> the file (uint8).  `document` = host numpy H x W x planes array; `layers` = ITW_PANE_2D:
        None or a list of (channels, alpha) as dds_encode_layers takes them; ITW_PANE_CUBE_LAYERS: six entries as cube_faces takes them;
        ignored for a cross."""
        doc = np.ascontiguousarray(document)
        n = self.none_layout(options, doc.shape[1], doc.shape[0])[0]
        if not n:
            raise ValueError("itw_dds_none_layout refused the options: " + self.last_error())
        keep, arr, count = [], None, 0
        if options.texture == PANE_CUBE_LAYERS:
            arr, count = self.cube_faces(layers, doc.dtype, keep), 6
        elif options.texture == PANE_2D and layers:
            arr, count = (LayerSource * len(layers))(), len(layers)
            for i, (channels, alpha) in enumerate(layers):
                one = self.cube_faces([(channels, alpha)], doc.dtype, keep)
                arr[i] = one[0]
        src = PixelSource(doc.ctypes.data, doc.shape[1], doc.shape[0], doc.shape[2], doc.itemsize * 8, 0)
        out = np.zeros(n, np.uint8)
        got = self.dds_save_none_raw(options, src, arr, count, flags, out.ctypes.data, n)
        if got != n:
            raise RuntimeError("itw_dds_save_none failed: " + self.last_error())
        return out

    def dds_save_none_raw(self, options, document, layers, count, flags, file_ptr, capacity):
        """itw_dds_save_none on ctypes structures (options and document may be None) and raw addresses; returns the file size (0 on error)."""
        f = self.lib.itw_dds_save_none
        f.restype = ctypes.c_size_t
        f.argtypes = [ctypes.POINTER(NoneOptions), ctypes.POINTER(PixelSource), ctypes.POINTER(LayerSource), ctypes.c_int, ctypes.c_uint32,
                      ctypes.c_void_p, ctypes.c_size_t]
        ref = lambda x: ctypes.byref(x) if x is not None else None
        return f(ref(options), ref(document), layers, count, flags, ctypes.c_void_p(file_ptr) if file_ptr else None, capacity)

    def dds_open(self, file_ptr, size):
        """itw_dds_open on a raw address (host or device): header + alpha check -> DdsOpenInfo."""
        f = self.lib.itw_dds_open
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsOpenInfo)]
        info = DdsOpenInfo()
        rc = f(ctypes.c_void_p(file_ptr), size, ctypes.byref(info))
        self.check()
        if rc != 0:
            raise RuntimeError("itw_dds_open failed")
        return info

    def dds_open_layout(self, info, options):
        """itw_dds_open_layout: fills the layout fields of `info` (in place) for the load dialog's answers `options`."""
        f = self.lib.itw_dds_open_layout
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(DdsOpenInfo), ctypes.c_uint32]
        rc = f(ctypes.byref(info), options)
        self.check()
        if rc != 0:
            raise RuntimeError("itw_dds_open_layout failed")
        return info

    def dds_read_layer_raw(self, file_ptr, size, info, call, dst_ptr, row_bytes=0):
        """itw_dds_read_layer on raw addresses (host or device)."""
        f = self.lib.itw_dds_read_layer
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsOpenInfo), ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
        rc = f(ctypes.c_void_p(file_ptr), size, ctypes.byref(info), call, ctypes.c_void_p(dst_ptr), row_bytes)
        self.check()
        if rc != 0:
            raise RuntimeError("itw_dds_read_layer failed")

    def dds_open_layers(self, file, options=0):
        """The plug-in's whole open path on a host DDS blob: (info, [layer arrays of height x width x planes, uint8 or float32])."""
        file = np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))
        info = self.dds_open_layout(self.dds_open(file.ctypes.data, file.size), options)
        layers = []
        for call in range(info.calls):
            out = np.empty((info.height, info.width, info.planes), np.float32 if info.depth == 32 else np.uint8)
            self.dds_read_layer_raw(file.ctypes.data, file.size, info, call, out.ctypes.data)
            layers.append(out)
        return info, layers

    def dds_open_uncompressed_raw(self, file_ptr, size, info):
        """itw_dds_open_uncompressed on a raw address (host or device) and a DdsUncompressedInfo (or None); returns its status."""
        f = self.lib.itw_dds_open_uncompressed
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsUncompressedInfo)]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None)

    def dds_open_uncompressed(self, file_ptr, size):
        """itw_dds_open_uncompressed: header + alpha check -> DdsUncompressedInfo."""
        info = DdsUncompressedInfo()
        if self.dds_open_uncompressed_raw(file_ptr, size, info) != 0:
            raise RuntimeError("itw_dds_open_uncompressed failed: " + self.last_error())
        return info

    def dds_uncompressed_layout_raw(self, info, options):
        f = self.lib.itw_dds_uncompressed_layout
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(DdsUncompressedInfo), ctypes.c_uint32]
        return f(ctypes.byref(info) if info is not None else None, options)

    def dds_uncompressed_layout(self, info, options):
        """itw_dds_uncompressed_layout: fills the layout fields of `info` (in place) for the load dialog's answers `options`."""
        if self.dds_uncompressed_layout_raw(info, options) != 0:
            raise RuntimeError("itw_dds_uncompressed_layout failed: " + self.last_error())
        return info

    def dds_read_uncompressed_layer_raw(self, file_ptr, size, info, call, dst_ptr, row_bytes=0):
        """itw_dds_read_uncompressed_layer on raw addresses (host or device); returns its status."""
        f = self.lib.itw_dds_read_uncompressed_layer
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsUncompressedInfo), ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None, call,
                 ctypes.c_void_p(dst_ptr) if dst_ptr else None, row_bytes)

    def dds_open_uncompressed_layers(self, file, options=0):
        """The plug-in's whole open path on a host uncompressed DDS blob: (info, [layer arrays of height x width x planes: uint8 at
        depth 8, uint16 at depth 16, float32 at depth 32])."""
        file = np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))
        info = self.dds_uncompressed_layout(self.dds_open_uncompressed(file.ctypes.data, file.size), options)
        dtype = {8: np.uint8, 16: np.uint16, 32: np.float32}[info.depth]
        layers = []
        for call in range(info.calls):
            out = np.empty((info.height, info.width, info.planes), dtype)
            if self.dds_read_uncompressed_layer_raw(file.ctypes.data, file.size, info, call, out.ctypes.data) != 0:
                raise RuntimeError("itw_dds_read_uncompressed_layer failed: " + self.last_error())
            layers.append(out)
        return info, layers

    def dds_open_converted_raw(self, file_ptr, size, info):
        """itw_dds_open_converted on a raw address (host or device) and a DdsConvertedInfo (or None); returns its status."""
        f = self.lib.itw_dds_open_converted
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsConvertedInfo)]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None)

    def dds_open_converted(self, file_ptr, size):
        """itw_dds_open_converted: header + alpha check -> DdsConvertedInfo."""
        info = DdsConvertedInfo()
        if self.dds_open_converted_raw(file_ptr, size, info) != 0:
            raise RuntimeError("itw_dds_open_converted failed: " + self.last_error())
        return info

    def dds_converted_layout_raw(self, info, options):
        f = self.lib.itw_dds_converted_layout
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(DdsConvertedInfo), ctypes.c_uint32]
        return f(ctypes.byref(info) if info is not None else None, options)

    def dds_converted_layout(self, info, options):
        """itw_dds_converted_layout: fills the layout fields of `info` (in place) for the load dialog's answers `options`."""
        if self.dds_converted_layout_raw(info, options) != 0:
            raise RuntimeError("itw_dds_converted_layout failed: " + self.last_error())
        return info

    def dds_read_converted_layer_raw(self, file_ptr, size, info, call, dst_ptr, row_bytes=0):
        """itw_dds_read_converted_layer on raw addresses (host or device); returns its status."""
        f = self.lib.itw_dds_read_converted_layer
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsConvertedInfo), ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None, call,
                 ctypes.c_void_p(dst_ptr) if dst_ptr else None, row_bytes)

    def dds_open_converted_layers(self, file, options=0):
        """The plug-in's whole open path on a host DDS blob it converts: (info, [layer arrays of height x width x planes: uint8 at
        depth 8, uint16 at depth 16, float32 at depth 32])."""
        file = np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))
        info = self.dds_converted_layout(self.dds_open_converted(file.ctypes.data, file.size), options)
        dtype = {8: np.uint8, 16: np.uint16, 32: np.float32}[info.depth]
        layers = []
        for call in range(info.calls):
            out = np.empty((info.height, info.width, info.planes), dtype)
            if self.dds_read_converted_layer_raw(file.ctypes.data, file.size, info, call, out.ctypes.data) != 0:
                raise RuntimeError("itw_dds_read_converted_layer failed: " + self.last_error())
            layers.append(out)
        return info, layers

    def dds_open_other_bc_raw(self, file_ptr, size, info):
        """itw_dds_open_other_bc on a raw address (host or device) and a DdsOtherBcInfo (or None); returns its status."""
        f = self.lib.itw_dds_open_other_bc
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsOtherBcInfo)]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None)

    def dds_open_other_bc(self, file_ptr, size):
        """itw_dds_open_other_bc: header + alpha check -> DdsOtherBcInfo."""
        info = DdsOtherBcInfo()
        if self.dds_open_other_bc_raw(file_ptr, size, info) != 0:
            raise RuntimeError("itw_dds_open_other_bc failed: " + self.last_error())
        return info

    def dds_other_bc_layout_raw(self, info, options):
        f = self.lib.itw_dds_other_bc_layout
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(DdsOtherBcInfo), ctypes.c_uint32]
        return f(ctypes.byref(info) if info is not None else None, options)

    def dds_other_bc_layout(self, info, options):
        """itw_dds_other_bc_layout: fills the layout fields of `info` (in place) for the load dialog's answers `options`."""
        if self.dds_other_bc_layout_raw(info, options) != 0:
            raise RuntimeError("itw_dds_other_bc_layout failed: " + self.last_error())
        return info

    def dds_read_other_bc_layer_raw(self, file_ptr, size, info, call, dst_ptr, row_bytes=0):
        """itw_dds_read_other_bc_layer on raw addresses (host or device); returns its status."""
        f = self.lib.itw_dds_read_other_bc_layer
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsOtherBcInfo), ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None, call,
                 ctypes.c_void_p(dst_ptr) if dst_ptr else None, row_bytes)

    def dds_open_other_bc_layers(self, file, options=0):
        """The plug-in's whole open path on a host DDS blob of the block-compressed formats itw_dds_open does not serve: (info,
        [layer arrays of height x width x planes: uint8 at depth 8, uint16 at depth 16])."""
        file = np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))
        info = self.dds_other_bc_layout(self.dds_open_other_bc(file.ctypes.data, file.size), options)
        dtype = {8: np.uint8, 16: np.uint16}[info.depth]
        layers = []
        for call in range(info.calls):
            out = np.empty((info.height, info.width, info.planes), dtype)
            if self.dds_read_other_bc_layer_raw(file.ctypes.data, file.size, info, call, out.ctypes.data) != 0:
                raise RuntimeError("itw_dds_read_other_bc_layer failed: " + self.last_error())
            layers.append(out)
        return info, layers

    def dds_open_expanded_raw(self, file_ptr, size, info):
        """itw_dds_open_expanded on a raw address (host or device) and a DdsExpandedInfo (or None); returns its status."""
        f = self.lib.itw_dds_open_expanded
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsExpandedInfo)]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None)

    def dds_open_expanded(self, file_ptr, size):
        """itw_dds_open_expanded: header + alpha check -> DdsExpandedInfo."""
        info = DdsExpandedInfo()
        if self.dds_open_expanded_raw(file_ptr, size, info) != 0:
            raise RuntimeError("itw_dds_open_expanded failed: " + self.last_error())
        return info

    def dds_expanded_layout_raw(self, info, options):
        f = self.lib.itw_dds_expanded_layout
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(DdsExpandedInfo), ctypes.c_uint32]
        return f(ctypes.byref(info) if info is not None else None, options)

    def dds_expanded_layout(self, info, options):
        """itw_dds_expanded_layout: fills the layout fields of `info` (in place) for the load dialog's answers `options`."""
        if self.dds_expanded_layout_raw(info, options) != 0:
            raise RuntimeError("itw_dds_expanded_layout failed: " + self.last_error())
        return info

    def dds_read_expanded_layer_raw(self, file_ptr, size, info, call, dst_ptr, row_bytes=0):
        """itw_dds_read_expanded_layer on raw addresses (host or device); returns its status."""
        f = self.lib.itw_dds_read_expanded_layer
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsExpandedInfo), ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None, call,
                 ctypes.c_void_p(dst_ptr) if dst_ptr else None, row_bytes)

    def dds_open_expanded_layers(self, file, options=0):
        """The plug-in's whole open path on a host P8 / A8P8 / A8R3G3B2 / A4L4 DDS blob: (info, [uint8 layer arrays of height x
        width x planes])."""
        file = np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))
        info = self.dds_expanded_layout(self.dds_open_expanded(file.ctypes.data, file.size), options)
        layers = []
        for call in range(info.calls):
            out = np.empty((info.height, info.width, info.planes), np.uint8)
            if self.dds_read_expanded_layer_raw(file.ctypes.data, file.size, info, call, out.ctypes.data) != 0:
                raise RuntimeError("itw_dds_read_expanded_layer failed: " + self.last_error())
            layers.append(out)
        return info, layers

    def dds_open_stack_raw(self, file_ptr, size, info):
        """itw_dds_open_stack on a raw address (host or device) and a DdsStackInfo (or None); returns its status."""
        f = self.lib.itw_dds_open_stack
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsStackInfo)]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None)

    def dds_open_stack(self, file_ptr, size):
        """itw_dds_open_stack: header + alpha check -> DdsStackInfo."""
        info = DdsStackInfo()
        if self.dds_open_stack_raw(file_ptr, size, info) != 0:
            raise RuntimeError("itw_dds_open_stack failed: " + self.last_error())
        return info

    def dds_stack_layout_raw(self, info, options):
        f = self.lib.itw_dds_stack_layout
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.POINTER(DdsStackInfo), ctypes.c_uint32]
        return f(ctypes.byref(info) if info is not None else None, options)

    def dds_stack_layout(self, info, options):
        """itw_dds_stack_layout: fills the layout fields of `info` (in place) for the load dialog's answers `options`."""
        if self.dds_stack_layout_raw(info, options) != 0:
            raise RuntimeError("itw_dds_stack_layout failed: " + self.last_error())
        return info

    def dds_read_stack_layer_raw(self, file_ptr, size, info, call, dst_ptr, row_bytes=0):
        """itw_dds_read_stack_layer on raw addresses (host or device); returns its status."""
        f = self.lib.itw_dds_read_stack_layer
        f.restype = ctypes.c_int
        f.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(DdsStackInfo), ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
        return f(ctypes.c_void_p(file_ptr) if file_ptr else None, size, ctypes.byref(info) if info is not None else None, call,
                 ctypes.c_void_p(dst_ptr) if dst_ptr else None, row_bytes)

    def dds_open_stack_layers(self, file, options=0):
        """The plug-in's whole open path on a host volume, 1-D or array DDS blob: (info, [layer arrays of height x width x planes,
        uint8 / uint16 / float32 by depth])."""
        file = np.ascontiguousarray(np.frombuffer(bytes(file), np.uint8))
        info = self.dds_stack_layout(self.dds_open_stack(file.ctypes.data, file.size), options)
        dtype = {8: np.uint8, 16: np.uint16, 32: np.float32}[info.depth]
        layers = []
        for call in range(info.calls):
            out = np.empty((info.height, info.width, info.planes), dtype)
            if self.dds_read_stack_layer_raw(file.ctypes.data, file.size, info, call, out.ctypes.data) != 0:
                raise RuntimeError("itw_dds_read_stack_layer failed: " + self.last_error())
            layers.append(out)
        return info, layers

    def check(self):
        e = self.last_error()
        if e:
            raise RuntimeError("libitw_bcn: " + e)

    def set_device(self, index):
        if self.lib.itw_set_device(int(index)) != 0:
            self.check()

    def set_devices(self, indices):
        """itw_set_devices: host -> host calls fan out over these GPUs (one process); [] = single-device behaviour."""
        arr = (ctypes.c_int * max(len(indices), 1))(*indices)
        self.lib.itw_set_devices.restype = ctypes.c_int
        self.lib.itw_set_devices.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.c_int]
        if self.lib.itw_set_devices(arr, len(indices)) != 0:
            self.check()
            raise RuntimeError("itw_set_devices failed")

    def begin_deferred(self):
        if self.lib.itw_begin_deferred() != 0:
            self.check()

    def flush(self):
        if self.lib.itw_flush() != 0:
            self.check()
            raise RuntimeError("itw_flush failed")

    def launch_count(self):
        return int(self.lib.itw_kernel_launch_count())

    def last_kernel_ms(self):
        return float(self.lib.itw_last_kernel_ms())

    def encode_batch(self, fmt, surfaces, dst_ptrs, settings=None):
        """itw_encode_batch: `surfaces` = list of (ptr, width, height, stride), `dst_ptrs` = list of addresses."""
        n = len(surfaces)
        arr = (RgbaSurface * n)(*[RgbaSurface(*s) for s in surfaces])
        dst = (ctypes.c_void_p * n)(*dst_ptrs)
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        self.lib.itw_encode_batch.argtypes = [ctypes.c_int, ctypes.POINTER(RgbaSurface), ctypes.POINTER(ctypes.c_void_p),
                                              ctypes.c_int, ctypes.c_void_p]
        if self.lib.itw_encode_batch(FORMATS[fmt][0], arr, dst, n, sp) != 0:
            self.check()
            raise RuntimeError("itw_encode_batch failed")

    def encode_device(self, fmt, ptr, width, height, stride, dst_ptr, settings=None, stream=0):
        """Enqueue the encode of a device-resident surface on a CUDA stream (no copies, no sync)."""
        surf = RgbaSurface(ptr, width, height, stride)
        sp = ctypes.cast(ctypes.byref(settings), ctypes.c_void_p) if settings is not None else None
        rc = self.lib.itw_encode_device(FORMATS[fmt][0], ctypes.byref(surf), ctypes.c_void_p(dst_ptr), sp,
                                        ctypes.c_void_p(stream))
        if rc != 0:
            self.check()
            raise RuntimeError("itw_encode_device failed")
