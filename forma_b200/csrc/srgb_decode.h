// The sRGB8 decode table of frames rendered over a background (forma_renderer_render_over_device):
// D[b] is the f32 nearest the standard sRGB EOTF of b / 255 when compute_srgb's encode
// (linear_to_srgb, to_byte) turns it back into b, and otherwise the f32 nearest that value among
// those it turns into b. Every byte round-trips. Bytes of the second kind: 11. The EOTF of
// 11 / 255 (0.0033465...) encodes to 12, because the encoder's polynomial branch reaches byte 11
// just above its linear branch's end at 0.0031308.
// Written by tools/make_srgb_decode.py with the oracle's encoder; tests/test_over_oracle.py pins it.
// Shared by the paint kernels (kernels_painter.cu) and the test oracle of frames over a background.
#pragma once

#define FORMA_SRGB_DECODE_TABLE \
    { \
    0x0.0p+0f, 0x1.3e4568p-12f, 0x1.3e4568p-11f, 0x1.dd681cp-11f, \
    0x1.3e4568p-10f, 0x1.8dd6c2p-10f, 0x1.dd681cp-10f, 0x1.167cbap-9f, \
    0x1.3e4568p-9f, 0x1.660e14p-9f, 0x1.8dd6c2p-9f, 0x1.b2a1b2p-9f, \
    0x1.e1e31ep-9f, 0x1.07c38cp-8f, 0x1.1fcc2cp-8f, 0x1.390ffap-8f, \
    0x1.53936cp-8f, 0x1.6f5adep-8f, 0x1.8c6a94p-8f, 0x1.aac6cp-8f, \
    0x1.ca7382p-8f, 0x1.eb74e2p-8f, 0x1.06e76cp-7f, 0x1.18c2a6p-7f, \
    0x1.2b4e0ap-7f, 0x1.3e8b7cp-7f, 0x1.527cd6p-7f, 0x1.6723eep-7f, \
    0x1.7c8292p-7f, 0x1.929a88p-7f, 0x1.a96d92p-7f, 0x1.c0fd68p-7f, \
    0x1.d94bbep-7f, 0x1.f25a44p-7f, 0x1.061552p-6f, 0x1.135f3ep-6f, \
    0x1.210bb8p-6f, 0x1.2f1b8cp-6f, 0x1.3d8f84p-6f, 0x1.4c6866p-6f, \
    0x1.5ba6fap-6f, 0x1.6b4c04p-6f, 0x1.7b5842p-6f, 0x1.8bcc74p-6f, \
    0x1.9ca958p-6f, 0x1.adefaap-6f, 0x1.bfa02p-6f, 0x1.d1bb74p-6f, \
    0x1.e4425ap-6f, 0x1.f73586p-6f, 0x1.054ad4p-5f, 0x1.0f31bap-5f, \
    0x1.194fccp-5f, 0x1.23a55ep-5f, 0x1.2e32c8p-5f, 0x1.38f86p-5f, \
    0x1.43f678p-5f, 0x1.4f2d64p-5f, 0x1.5a9d76p-5f, 0x1.664702p-5f, \
    0x1.722a56p-5f, 0x1.7e47c8p-5f, 0x1.8a9fa4p-5f, 0x1.97323ap-5f, \
    0x1.a3ffd8p-5f, 0x1.b108dp-5f, 0x1.be4d6cp-5f, 0x1.cbcdfap-5f, \
    0x1.d98ac6p-5f, 0x1.e7841cp-5f, 0x1.f5ba48p-5f, 0x1.0216cap-4f, \
    0x1.096f26p-4f, 0x1.10e65cp-4f, 0x1.187c9p-4f, 0x1.2031e8p-4f, \
    0x1.280688p-4f, 0x1.2ffa92p-4f, 0x1.380e2ap-4f, 0x1.404174p-4f, \
    0x1.489494p-4f, 0x1.5107acp-4f, 0x1.599adep-4f, 0x1.624e4ep-4f, \
    0x1.6b221ep-4f, 0x1.74167p-4f, 0x1.7d2b66p-4f, 0x1.86612p-4f, \
    0x1.8fb7cp-4f, 0x1.992f68p-4f, 0x1.a2c83ap-4f, 0x1.ac8256p-4f, \
    0x1.b65ddcp-4f, 0x1.c05aecp-4f, 0x1.ca79a8p-4f, 0x1.d4ba3p-4f, \
    0x1.df1ca2p-4f, 0x1.e9a12p-4f, 0x1.f447cap-4f, 0x1.ff10bcp-4f, \
    0x1.04fe0cp-3f, 0x1.0a84fep-3f, 0x1.101d44p-3f, 0x1.15c6eep-3f, \
    0x1.1b8208p-3f, 0x1.214ea6p-3f, 0x1.272cd4p-3f, 0x1.2d1ca2p-3f, \
    0x1.331e1ep-3f, 0x1.393158p-3f, 0x1.3f566p-3f, 0x1.458d42p-3f, \
    0x1.4bd60ep-3f, 0x1.5230d4p-3f, 0x1.589dap-3f, 0x1.5f1c84p-3f, \
    0x1.65ad8ap-3f, 0x1.6c50c4p-3f, 0x1.73063ep-3f, 0x1.79ce06p-3f, \
    0x1.80a82ep-3f, 0x1.8794cp-3f, 0x1.8e93ccp-3f, 0x1.95a55ep-3f, \
    0x1.9cc986p-3f, 0x1.a40052p-3f, 0x1.ab49cep-3f, 0x1.b2a60ap-3f, \
    0x1.ba1512p-3f, 0x1.c196f4p-3f, 0x1.c92bbep-3f, 0x1.d0d37cp-3f, \
    0x1.d88e3ep-3f, 0x1.e05c0ep-3f, 0x1.e83cfcp-3f, 0x1.f03116p-3f, \
    0x1.f83866p-3f, 0x1.00297ep-2f, 0x1.044072p-2f, 0x1.086116p-2f, \
    0x1.0c8b7p-2f, 0x1.10bf86p-2f, 0x1.14fd6p-2f, 0x1.194502p-2f, \
    0x1.1d9676p-2f, 0x1.21f1bep-2f, 0x1.2656e4p-2f, 0x1.2ac5ecp-2f, \
    0x1.2f3edep-2f, 0x1.33c1cp-2f, 0x1.384e98p-2f, 0x1.3ce56cp-2f, \
    0x1.418642p-2f, 0x1.46312p-2f, 0x1.4ae60ep-2f, 0x1.4fa51p-2f, \
    0x1.546e2cp-2f, 0x1.59416cp-2f, 0x1.5e1edp-2f, 0x1.630664p-2f, \
    0x1.67f82ap-2f, 0x1.6cf428p-2f, 0x1.71fa68p-2f, 0x1.770aecp-2f, \
    0x1.7c25bcp-2f, 0x1.814adcp-2f, 0x1.867a54p-2f, 0x1.8bb428p-2f, \
    0x1.90f86p-2f, 0x1.9647p-2f, 0x1.9ba01p-2f, 0x1.a10394p-2f, \
    0x1.a67192p-2f, 0x1.abea1p-2f, 0x1.b16d14p-2f, 0x1.b6faa4p-2f, \
    0x1.bc92c6p-2f, 0x1.c2357ep-2f, 0x1.c7e2d2p-2f, 0x1.cd9acap-2f, \
    0x1.d35d6ap-2f, 0x1.d92ab6p-2f, 0x1.df02b8p-2f, 0x1.e4e57p-2f, \
    0x1.ead2e8p-2f, 0x1.f0cb26p-2f, 0x1.f6ce2cp-2f, 0x1.fcdcp-2f, \
    0x1.017a56p-1f, 0x1.048c18p-1f, 0x1.07a34ap-1f, 0x1.0abfeep-1f, \
    0x1.0de208p-1f, 0x1.11099ap-1f, 0x1.1436a8p-1f, 0x1.176932p-1f, \
    0x1.1aa13ep-1f, 0x1.1ddecap-1f, 0x1.2121dep-1f, 0x1.246a7ap-1f, \
    0x1.27b8ap-1f, 0x1.2b0c54p-1f, 0x1.2e6598p-1f, 0x1.31c46ep-1f, \
    0x1.3528dcp-1f, 0x1.3892ep-1f, 0x1.3c028p-1f, 0x1.3f77bcp-1f, \
    0x1.42f29ap-1f, 0x1.467318p-1f, 0x1.49f93ep-1f, 0x1.4d850ap-1f, \
    0x1.511682p-1f, 0x1.54ada4p-1f, 0x1.584a78p-1f, 0x1.5becfep-1f, \
    0x1.5f9538p-1f, 0x1.634328p-1f, 0x1.66f6d4p-1f, 0x1.6ab03ap-1f, \
    0x1.6e6f6p-1f, 0x1.723448p-1f, 0x1.75fef4p-1f, 0x1.79cf64p-1f, \
    0x1.7da59ep-1f, 0x1.8181a4p-1f, 0x1.856378p-1f, 0x1.894b1cp-1f, \
    0x1.8d3892p-1f, 0x1.912bdep-1f, 0x1.9525p-1f, 0x1.9923fep-1f, \
    0x1.9d28d8p-1f, 0x1.a13392p-1f, 0x1.a5442cp-1f, 0x1.a95aacp-1f, \
    0x1.ad771p-1f, 0x1.b1995ep-1f, 0x1.b5c198p-1f, 0x1.b9efbep-1f, \
    0x1.be23d4p-1f, 0x1.c25ddep-1f, 0x1.c69ddcp-1f, 0x1.cae3d2p-1f, \
    0x1.cf2fcp-1f, 0x1.d381aap-1f, 0x1.d7d994p-1f, 0x1.dc377ep-1f, \
    0x1.e09b6ap-1f, 0x1.e5055cp-1f, 0x1.e97556p-1f, 0x1.edeb5cp-1f, \
    0x1.f2676cp-1f, 0x1.f6e98cp-1f, 0x1.fb71bcp-1f, 0x1.0p+0f, \
    }
