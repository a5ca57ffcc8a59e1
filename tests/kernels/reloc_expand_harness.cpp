// Host build of the relocalisation grid (fast_lio_b200/csrc/reloc.cuh, the formula k_reloc_expand runs): reads the prior (26
// doubles), the grid's counts (4 ints) and steps (4 doubles) from stdin and writes the hypotheses ([H][26] doubles) to stdout.
#include <cstdio>
#include <vector>

#include "../../fast_lio_b200/csrc/reloc.cuh"

int main() {
    double prior[26];
    fl_reloc_grid_t g;
    if (fread(prior, sizeof(double), 26, stdin) != 26 || fread(g.n, sizeof(int), 4, stdin) != 4 || fread(g.step, sizeof(double), 4, stdin) != 4)
        return 1;
    const long long H = (long long)g.n[0] * g.n[1] * g.n[2] * g.n[3];
    std::vector<double> out(26 * (size_t)H);
    for (long long h = 0; h < H; h++)
        for (int c = 0; c < 26; c++) out[26 * (size_t)h + c] = fl::reloc_component(prior, g, h, c);
    return fwrite(out.data(), sizeof(double), out.size(), stdout) == out.size() ? 0 : 2;
}
