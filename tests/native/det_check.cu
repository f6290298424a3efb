// Host-side check of the fixed-point helpers of deterministic mode (dreamscene_b200/csrc/common.cuh).
// Built with nvcc and run on the CPU by tests/test_deterministic_cpu.py (no GPU needed).
#include <cmath>
#include <cstdio>
#include <cstring>
#include "common.cuh"

static int fails = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++fails; } } while (0)

static uint32_t bits(float x) { uint32_t u; std::memcpy(&u, &x, 4); return u; }
static float from_bits(uint32_t u) { float x; std::memcpy(&x, &u, 4); return x; }

int main() {
    const double K = GSR_DET_FIX_BITS;
    // round trip of one partial: error <= 2^-K of the component's largest |partial|
    const float maxima[] = {1.0f, 3.0e-8f, 7.5e5f, 1.0e-38f, 1.0e-44f, 3.0e38f, 0.0f};
    for (float mx : maxima) {
        const uint32_t mb = bits(std::fabs(mx));
        const int s = gsr_det_shift(mb);
        const float parts[] = {mx, -mx, 0.5f * mx, 0.3333f * mx, -0.7071f * mx, from_bits(mb == 0 ? 0u : mb - 1)};
        for (float x : parts) {
            const long long q = gsr_det_quantise(x, s);
            CHECK(std::llabs(q) <= (1ll << (GSR_DET_FIX_BITS + 1)));          // |partial| * 2^s <= 2^(K+1)
            const double back = (double)gsr_det_dequantise(q, mb);
            CHECK(std::fabs(back - (double)x) <= std::ldexp((double)std::fabs(mx), -(int)K) + std::ldexp(std::fabs((double)x), -24));
        }
    }
    // headroom: the largest number of commits one Gaussian can receive (8 per tile of its view), every one of
    // them the largest magnitude the component allows, sums without overflow and dequantises exactly
    const long long ncommits = 8ll * GSR_DET_MAX_VIEW_TILES;
    CHECK(ncommits == (1ll << 21));
    const float worst = from_bits(0x3fffffffu);                                // just below 2.0: largest mantissa
    const uint32_t wb = bits(worst);
    const long long qw = gsr_det_quantise(worst, gsr_det_shift(wb));
    CHECK(qw > 0 && qw <= (1ll << (GSR_DET_FIX_BITS + 1)));
    CHECK(qw <= INT64_MAX / ncommits);                                          // no signed overflow
    unsigned long long acc = 0ull;                                              // two's-complement, as atomicAdd
    for (long long k = 0; k < ncommits; ++k) acc += (unsigned long long)qw;
    CHECK((long long)acc > 0 && (long long)acc == qw * ncommits);
    const double sum = (double)gsr_det_dequantise((long long)acc, wb);
    CHECK(std::fabs(sum - (double)worst * (double)ncommits) <= 1e-6 * (double)worst * (double)ncommits);
    // opposite signs cancel exactly in any order
    const long long qa = gsr_det_quantise(0.625f, gsr_det_shift(bits(1.5f)));
    const long long qb = gsr_det_quantise(-0.625f, gsr_det_shift(bits(1.5f)));
    CHECK(qa + qb == 0);
    // NaN and Inf partials make the component non-finite (never a finite wrong value)
    CHECK(!gsr_det_finite(bits(std::fabs(NAN))) && !gsr_det_finite(bits(INFINITY)) && gsr_det_finite(bits(3.0e38f)));
    CHECK(std::isnan(gsr_det_dequantise(0, bits(std::fabs(NAN)))));
    CHECK(std::isnan(gsr_det_dequantise(12345, bits(INFINITY))));
    // important score: fixed scale, a view's worth of full-weight pixels fits, a small weight survives
    const long long pixels = (long long)GSR_DET_MAX_VIEW_TILES * GSR_TILE * GSR_TILE;
    const long long q32 = gsr_det_score_quantise(32.0f);                        // one warp, every pixel weight 1
    CHECK(q32 <= INT64_MAX / (pixels / 32));
    CHECK(gsr_det_score_dequantise(q32 * (pixels / 32)) == (float)pixels);
    const float w = 4.0e-7f;                                                     // alpha_min * T_stop
    CHECK(std::fabs((double)gsr_det_score_dequantise(gsr_det_score_quantise(w)) - (double)w) <= std::ldexp(1.0, -GSR_DET_SCORE_BITS));
    std::printf(fails ? "%d checks failed\n" : "deterministic helpers ok\n", fails);
    return fails ? 1 : 0;
}
