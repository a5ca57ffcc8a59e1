// The partial row of the wave kernels (k_update_wave, k_update_n_wave and their _det twins): which of the 96 sums of a
// k_update partial row (PSTRIDE: the 12-wide upper triangle of H^T H, H^T h, effct, sum |res|, pads) each slot carries.
// With extrinsic estimation warp_accumulate writes 92 of the 96 entries, and the row is the whole 96.  Without it, it writes
// only 29 -- the 21 entries of H^T H with a <= b < 6, H^T h[0..5], effct and sum |res| -- and the other 67 are +0.0 in every
// row of every pass, so the row is 32 doubles: slots 0..20 the a <= b < 6 pairs in warp_accumulate's order (row-major), 21..26
// H^T h, 27 effct, 28 sum |res|, 29..31 +0.0 pads.  Each slot is summed exactly as its entry is in k_update, and an entry no
// slot carries is +0.0 there, so the solver's 96 sums keep k_update's bits.  Host and device: tests compile this header alone.
#pragma once

namespace fl {

template <bool EXTR> struct WaveRow {
    static constexpr int W = EXTR ? 96 : 32;       // doubles per row
    static constexpr int LIVE = EXTR ? 96 : 29;     // slots that carry an entry
};

// the entry of the 96 sums that slot s of the row carries (s < WaveRow<EXTR>::LIVE)
template <bool EXTR>
__host__ __device__ constexpr int wave_entry(int s) {
    if (EXTR) return s;
    if (s < 21) {
        int a = 0, rem = s;
        while (rem >= 6 - a) { rem -= 6 - a; a++; }
        return a * 12 - (a * (a - 1)) / 2 + rem;     // (a, b = a + rem) in the 12-wide triangle
    }
    return s < 27 ? 78 + (s - 21) : 90 + (s - 27);
}

// the slot that carries entry o of the 96 sums, or -1 if none (an entry that is +0.0 in every row)
template <bool EXTR>
__host__ __device__ constexpr int wave_slot(int o) {
    for (int s = 0; s < WaveRow<EXTR>::LIVE; s++)
        if (wave_entry<EXTR>(s) == o) return s;
    return -1;
}

static_assert(wave_entry<false>(20) == 5 * 12 - 10 + 0 && wave_slot<false>(90) == 27 && wave_slot<false>(91) == 28 &&
                  wave_slot<false>(6) == -1 && wave_slot<false>(84) == -1 && wave_slot<true>(90) == 90,
              "the compact row's index map");

}  // namespace fl
