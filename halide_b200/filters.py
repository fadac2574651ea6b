"""Python call sites of the C-ABI filters, one function per exported symbol.

Same names, argument order and error behaviour as the generated AOT functions the reference's
harnesses call (apps/*/process.cpp, apps/blur/test.cpp): a negative halide_error_code_t becomes a
:class:`HalideError`.  Outputs are left device-dirty, exactly like a Halide GPU filter; call
``out.copy_to_host()`` to read them on the host.
"""
import ctypes

from .lib import lib, check


def halide_blur(input, blur_y):
    """apps/blur/halide_blur_generator.cpp: 3x3 box filter, uint16."""
    return check(lib.halide_blur(input.ptr, blur_y.ptr))


def local_laplacian(input, levels, alpha, beta, output):
    """apps/local_laplacian/local_laplacian_generator.cpp.  NOTE: like the harness
    (process.cpp:31) callers pass alpha already divided by (levels - 1)."""
    return check(lib.local_laplacian(input.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                     ctypes.c_float(beta), output.ptr))


def local_laplacian_batch(input, levels, alpha, beta, output):
    """local_laplacian on every frame of 4-D (x, y, c, n) buffers, e.g. an (N, 3, H, W) uint16 torch tensor or numpy
    array: output frame n = local_laplacian(input frame n), bit for bit, in one launch sequence for the whole batch."""
    return check(lib.halide_b200_local_laplacian_batch(input.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                                       ctypes.c_float(beta), output.ptr))


def local_laplacian_u8(input, levels, alpha, beta, output):
    """local_laplacian on 3-D (x, y, c) uint8 buffers: output = to_u8(local_laplacian(to_u16(input))) bit for bit, with the
    reference's element conversions (image_io.convert: to_u16(v) = v * 257, to_u8(w) = ((w + 128) * 255 + 255) >> 16),
    done inside the kernels: no uint16 copy of either frame is made."""
    return check(lib.halide_b200_local_laplacian_u8(input.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                                    ctypes.c_float(beta), output.ptr))


def local_laplacian_u8_batch(input, levels, alpha, beta, output):
    """local_laplacian_u8 on every frame of 4-D (x, y, c, n) uint8 buffers, e.g. an (N, 3, H, W) uint8 torch tensor (a
    decoded clip): output frame n = local_laplacian_u8(input frame n), in one launch sequence for the whole batch."""
    return check(lib.halide_b200_local_laplacian_u8_batch(input.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                                          ctypes.c_float(beta), output.ptr))


def local_laplacian_pyramid_levels(input, pyramid_levels, levels, alpha, beta, output):
    """local_laplacian with the generator's pyramid_levels J (the pyramid depth: the coarsest level's pixels cover 2^(J-1)
    frame pixels, the spatial scale of the detail the filter manipulates) chosen per call, 1 <= J <= 20: the result is
    what the generator built with that J computes, bit for bit.  Buffers (3-D uint16), levels, alpha, beta and error
    codes as local_laplacian; J = 8 is local_laplacian itself."""
    return check(lib.halide_b200_local_laplacian_pyramid_levels(input.ptr, ctypes.c_int32(pyramid_levels), ctypes.c_int32(levels),
                                                                ctypes.c_float(alpha), ctypes.c_float(beta), output.ptr))


_INTERLEAVED_LAYOUT = """
    Both buffers are pixel-interleaved (RGBRGB..., RGBA...): ``dim[2].stride == 1`` and ``dim[0].stride`` is the pixel
    pitch, at least the channel extent; ``dim[1].stride`` (and ``dim[3].stride``) positive.  Anything else, a planar
    buffer included, is refused with -8.  The result is, bit for bit, what the planar entry point gives on planar copies
    of the same buffers.  An output whose pitch exceeds its channel extent (channels [0, 3) of an RGBA frame) leaves the
    samples it does not cover untouched.  The common sources:

    - a torch tensor in ``torch.channels_last`` memory format: ``HalideBuffer.from_torch(t)`` already describes it as
      ``(x: C, y: W*C, c: 1, n: H*W*C)``;
    - a numpy ``(H, W, C)`` array (PIL, OpenCV): ``HalideBuffer.from_numpy(arr.transpose(2, 0, 1))``.
    """


def local_laplacian_interleaved(input, levels, alpha, beta, output):
    return check(lib.halide_b200_local_laplacian_interleaved(input.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                                             ctypes.c_float(beta), output.ptr))


def local_laplacian_interleaved_batch(input, levels, alpha, beta, output):
    return check(lib.halide_b200_local_laplacian_interleaved_batch(input.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                                                   ctypes.c_float(beta), output.ptr))


def local_laplacian_u8_interleaved(input, levels, alpha, beta, output):
    return check(lib.halide_b200_local_laplacian_u8_interleaved(input.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                                                ctypes.c_float(beta), output.ptr))


def local_laplacian_u8_interleaved_batch(input, levels, alpha, beta, output):
    return check(lib.halide_b200_local_laplacian_u8_interleaved_batch(input.ptr, ctypes.c_int32(levels), ctypes.c_float(alpha),
                                                                      ctypes.c_float(beta), output.ptr))


local_laplacian_interleaved.__doc__ = "local_laplacian on 3-D (x, y, c) uint16 interleaved buffers.\n" + _INTERLEAVED_LAYOUT
local_laplacian_interleaved_batch.__doc__ = ("local_laplacian_batch on 4-D (x, y, c, n) uint16 interleaved buffers, e.g. an "
                                             "(N, 3, H, W) channels_last tensor.\n" + _INTERLEAVED_LAYOUT)
local_laplacian_u8_interleaved.__doc__ = "local_laplacian_u8 on 3-D (x, y, c) uint8 interleaved buffers.\n" + _INTERLEAVED_LAYOUT
local_laplacian_u8_interleaved_batch.__doc__ = ("local_laplacian_u8_batch on 4-D (x, y, c, n) uint8 interleaved buffers, e.g. a "
                                                "decoded (N, 3, H, W) channels_last clip.\n" + _INTERLEAVED_LAYOUT)


def stencil_chain(input, output):
    """apps/stencil_chain/stencil_chain_generator.cpp: 32 chained 5x5 uint16 stencils."""
    return check(lib.stencil_chain(input.ptr, output.ptr))


def stencil_chain_stencils(input, stencils, output):
    """stencil_chain with the generator's stencils (the number of chained 5x5 stages, the depth of the chain and so the
    reach of the filter: 2 * stencils px each way) chosen per call, 1 <= stencils <= 100: the result is what the generator
    built with that stencils computes, bit for bit.  Buffers and error codes as stencil_chain; stencils = 32 is
    stencil_chain itself."""
    return check(lib.halide_b200_stencil_chain_stencils(input.ptr, ctypes.c_int32(stencils), output.ptr))


def bilateral_grid(input, r_sigma, output):
    """apps/bilateral_grid/bilateral_grid_generator.cpp (s_sigma = 8), float32."""
    return check(lib.bilateral_grid(input.ptr, ctypes.c_float(r_sigma), output.ptr))


def bilateral_grid_s_sigma(input, s_sigma, r_sigma, output):
    """bilateral_grid with the generator's s_sigma (grid cell size in pixels, the spatial scale of the smoothing) chosen
    per call, 1 <= s_sigma <= 128: the result is what the generator built with that s_sigma computes.  Buffers, r_sigma
    and error codes as bilateral_grid; s_sigma = 8 is bilateral_grid itself, bit for bit."""
    return check(lib.halide_b200_bilateral_grid_s_sigma(input.ptr, ctypes.c_int32(s_sigma), ctypes.c_float(r_sigma),
                                                        output.ptr))


def nl_means(input, patch_size, search_area, sigma, output):
    """apps/nl_means/nl_means_generator.cpp, float32, output has exactly 3 channels."""
    return check(lib.nl_means(input.ptr, ctypes.c_int32(patch_size), ctypes.c_int32(search_area),
                              ctypes.c_float(sigma), output.ptr))


_U8_CONVERSIONS = """

    The conversions are the reference's image I/O (image_io.convert): to_f32(v) = v / 255.0f, an IEEE float division, and
    to_u8(f) = lround(f * 255.0f), the product rounded to float32 and then to the nearest integer with halves away from
    zero.  Both run inside the kernels that read and write the frame: no float copy of either frame is made."""


def bilateral_grid_u8(input, r_sigma, output):
    return check(lib.halide_b200_bilateral_grid_u8(input.ptr, ctypes.c_float(r_sigma), output.ptr))


def nl_means_u8(input, patch_size, search_area, sigma, output):
    return check(lib.halide_b200_nl_means_u8(input.ptr, ctypes.c_int32(patch_size), ctypes.c_int32(search_area),
                                             ctypes.c_float(sigma), output.ptr))


bilateral_grid_u8.__doc__ = ("bilateral_grid on 2-D (x, y) uint8 buffers, e.g. an (H, W) uint8 torch tensor:\n"
                             "output = to_u8(bilateral_grid(to_f32(input), r_sigma)) byte for byte.  Buffer rules and error "
                             "codes as bilateral_grid." + _U8_CONVERSIONS)
nl_means_u8.__doc__ = ("nl_means on 3-D (x, y, c) uint8 buffers, e.g. a (3, H, W) uint8 torch tensor:\n"
                       "output = to_u8(nl_means(to_f32(input), patch_size, search_area, sigma)) byte for byte.  Buffer "
                       "rules (output channels exactly [0, 3)) and error codes as nl_means." + _U8_CONVERSIONS)


def camera_pipe(input, matrix_3200, matrix_7000, color_temp, gamma, contrast, sharpen_strength, blackLevel, whiteLevel,
                processed):
    """apps/camera_pipe/camera_pipe_generator.cpp: uint16 Bayer raw -> uint8 RGB."""
    return check(lib.camera_pipe(input.ptr, matrix_3200.ptr, matrix_7000.ptr, ctypes.c_float(color_temp),
                                 ctypes.c_float(gamma), ctypes.c_float(contrast), ctypes.c_float(sharpen_strength),
                                 ctypes.c_int32(blackLevel), ctypes.c_int32(whiteLevel), processed.ptr))


def _camera_pipe_scalars(color_temp, gamma, contrast, sharpen_strength, blackLevel, whiteLevel):
    return (ctypes.c_float(color_temp), ctypes.c_float(gamma), ctypes.c_float(contrast), ctypes.c_float(sharpen_strength),
            ctypes.c_int32(blackLevel), ctypes.c_int32(whiteLevel))


def camera_pipe_batch(input, matrix_3200, matrix_7000, color_temp, gamma, contrast, sharpen_strength, blackLevel,
                      whiteLevel, processed):
    """camera_pipe on every frame of a raw burst, in one launch: input (x, y, n), e.g. an (N, H, W) uint16 tensor, and a
    planar output (x, y, c, n), e.g. an (N, 3, H, W) uint8 tensor.  Output frame n is camera_pipe(input frame n) byte for
    byte; the matrices and scalars are shared by all frames.  The input must cover the raw region camera_pipe needs and
    the output's frames, else -4."""
    return check(lib.halide_b200_camera_pipe_batch(input.ptr, matrix_3200.ptr, matrix_7000.ptr,
                                                   *_camera_pipe_scalars(color_temp, gamma, contrast, sharpen_strength,
                                                                         blackLevel, whiteLevel), processed.ptr))


_CAMERA_PIPE_INTERLEAVED = """
    The output is pixel-interleaved (RGBRGB..., RGBA...): ``dim[2].stride == 1``, ``dim[0].stride`` is the pixel pitch, at
    least the channel extent, and ``dim[1].stride`` (and ``dim[3].stride``) positive; anything else, a planar buffer
    included, is refused with -8.  The bytes are those the planar entry point writes, transposed; samples the output's
    channels do not cover (the alpha of an RGBA frame) are left untouched.  The common outputs:

    - an ``(N, H, W, 3)`` uint8 tensor (torchvision's video layout) passed as ``t.permute(0, 3, 1, 2)``, or an
      ``(N, 3, H, W)`` tensor in ``torch.channels_last`` memory format, which ``HalideBuffer.from_torch`` already
      describes as interleaved;
    - a numpy ``(H, W, 3)`` array (PIL, OpenCV, image encoders): ``HalideBuffer.from_numpy(arr.transpose(2, 0, 1))``.
    """


def camera_pipe_interleaved(input, matrix_3200, matrix_7000, color_temp, gamma, contrast, sharpen_strength, blackLevel,
                            whiteLevel, processed):
    return check(lib.halide_b200_camera_pipe_interleaved(input.ptr, matrix_3200.ptr, matrix_7000.ptr,
                                                         *_camera_pipe_scalars(color_temp, gamma, contrast, sharpen_strength,
                                                                               blackLevel, whiteLevel), processed.ptr))


def camera_pipe_interleaved_batch(input, matrix_3200, matrix_7000, color_temp, gamma, contrast, sharpen_strength,
                                  blackLevel, whiteLevel, processed):
    return check(lib.halide_b200_camera_pipe_interleaved_batch(input.ptr, matrix_3200.ptr, matrix_7000.ptr,
                                                               *_camera_pipe_scalars(color_temp, gamma, contrast,
                                                                                     sharpen_strength, blackLevel,
                                                                                     whiteLevel), processed.ptr))


camera_pipe_interleaved.__doc__ = ("camera_pipe into a 3-D (x, y, c) uint8 interleaved output; the raw input is camera_pipe's "
                                   "(H, W) uint16 frame.\n" + _CAMERA_PIPE_INTERLEAVED)
camera_pipe_interleaved_batch.__doc__ = ("camera_pipe_batch into a 4-D (x, y, c, n) uint8 interleaved output: a raw burst, an "
                                         "(N, H, W) uint16 tensor, to (N, H, W, 3) RGB in one launch.\n" +
                                         _CAMERA_PIPE_INTERLEAVED)


def conv_layer(input, filter, bias, relu):
    """apps/conv_layer/conv_layer_generator.cpp: 3x3 conv + bias + relu, fixed shapes (N5 CI128 CO128 100x80), f32."""
    return check(lib.conv_layer(input.ptr, filter.ptr, bias.ptr, relu.ptr))


def conv_layer_any_shape(input, filter, bias, relu):
    """conv_layer (3x3 conv + bias + relu, f32) with N, CI, CO, W and H taken from the buffers instead of the generator's
    fixed shape: relu (co, x, y, n) gives CO, W, H, N and the mins, filter (co, kx, ky, ci) gives CI; input (ci, x, y, n)
    must cover the output's region grown by two columns and two rows (the caller pads; nothing is clamped), filter and
    bias the output's channels, else -4.  Buffers may be larger than required and every stride but the channel one (1,
    else -8) is free, so crops and padded rows of larger tensors work in place.  In torch terms: an NHWC input
    ``[N, H + 2, W + 2, CI]``, a filter ``[CI, 3, 3, CO]``, a bias ``[CO]`` and an NHWC output ``[N, H, W, CO]``.  At
    conv_layer's shape the result is conv_layer's, byte for byte."""
    return check(lib.halide_b200_conv_layer_any_shape(input.ptr, filter.ptr, bias.ptr, relu.ptr))
