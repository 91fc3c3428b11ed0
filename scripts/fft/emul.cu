// emul.cu -- runs the per-thread phases of fftcore.cuh thread-by-thread on the CPU and compares with a float64 DFT.
//   nvcc -O2 -std=c++17 -I passiveradar_b200/csrc -o /tmp/fft_emul scripts/fft/emul.cu && /tmp/fft_emul
//   /tmp/fft_emul seeds      frame_pass_kernel's twiddle source (Tw1Seeds, R3 = 8) against the table: one key=value line
//   /tmp/fft_emul rows       frame_pass_kernel's pass-2 twiddle rows (Tw2Rows, R3 = 8): their values, the banks of their
//                            loads, and whole transforms against the tw2 table: one key=value line
// No CUDA runtime call is made: this pins the index algebra / twiddle conventions without a GPU.
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdio>
#include <random>
#include <string>
#include <vector>
#include "fftcore.cuh"

using namespace prc::fft;
typedef std::complex<double> cd;

template <int R3>
void make_tw(std::vector<float2>& tw) {
    using G = Geo<R3>;
    tw.resize(G::TW1 + G::TW2);
    for (int i = 0; i < G::TW1; ++i) {
        const int k1 = i / G::T, t = i % G::T;
        const double a = -2.0 * M_PI * (double)((long long)t * k1 % G::L) / G::L;
        tw[i] = make_float2((float)cos(a), (float)sin(a));
    }
    for (int q = 0; q < G::TW2; ++q) {
        const int k2 = q / R3, n3 = q % R3;
        const double a = -2.0 * M_PI * (double)(n3 * k2) / (16 * R3);
        tw[G::TW1 + q] = make_float2((float)cos(a), (float)sin(a));
    }
}

template <int R3>
int run() {
    using G = Geo<R3>;
    std::mt19937 rng(1234 + R3);
    std::normal_distribution<float> nd;
    std::vector<float2> x(G::L), tw;
    for (auto& v : x) v = make_float2(nd(rng), nd(rng));
    make_tw<R3>(tw);
    const float2* tw1 = tw.data();
    const float2* tw2 = tw.data() + G::TW1;
    std::vector<float2> ea(G::EX), eb(G::EX);
    struct Regs { float2 v[16]; };
    std::vector<Regs> regs(G::T);
    // float64 DFT
    std::vector<cd> X(G::L);
    for (int k = 0; k < G::L; ++k) {
        cd s = 0;
        for (int n = 0; n < G::L; ++n) {
            const double a = -2.0 * M_PI * (double)((long long)n * k % G::L) / G::L;
            s += cd(x[n].x, x[n].y) * cd(cos(a), sin(a));
        }
        X[k] = s;
    }
    double xmax = 0;
    for (auto& v : X) xmax = std::max(xmax, std::abs(v));
    // n2p
    for (int t = 0; t < G::T; ++t) for (int n1 = 0; n1 < 16; ++n1) regs[t].v[n1] = x[n1 * G::T + t];
    for (int t = 0; t < G::T; ++t) n2p_pass1<R3>(regs[t].v, t, ea.data(), Tw1Table<R3>{tw1});
    for (int t = 0; t < G::T; ++t) n2p_pass2<R3>(regs[t].v, t, ea.data(), eb.data(), Tw2Table<R3>{tw2});
    for (int t = 0; t < G::T; ++t) n2p_pass3<R3>(regs[t].v, t, eb.data());
    double e1 = 0;
    std::vector<int> seen(G::L, 0);
    for (int t = 0; t < G::T; ++t)
        for (int r = 0; r < 16; ++r) {
            const int f = perm_freq<R3>(t, r);
            seen[f]++;
            e1 = std::max(e1, std::abs(cd(regs[t].v[r].x, regs[t].v[r].y) - X[f]));
        }
    int bad = 0;
    for (int f = 0; f < G::L; ++f) bad += seen[f] != 1;
    // p2n applied to the permuted spectrum: y[n] = sum_k X[k] W^{nk}  ==  L * x[(-n) mod L]
    for (int t = 0; t < G::T; ++t) p2n_pass1<R3>(regs[t].v, t, eb.data());
    for (int t = 0; t < G::T; ++t) p2n_pass2<R3>(regs[t].v, t, eb.data(), ea.data(), Tw2Table<R3>{tw2});
    for (int t = 0; t < G::T; ++t) p2n_pass3<R3>(regs[t].v, t, ea.data(), Tw1Table<R3>{tw1});
    double e2 = 0, ymax = 0;
    for (int t = 0; t < G::T; ++t)
        for (int n1 = 0; n1 < 16; ++n1) {
            const int n = n1 * G::T + t;
            const float2 want = x[(G::L - n) % G::L];
            const cd w((double)want.x * G::L, (double)want.y * G::L);
            ymax = std::max(ymax, std::abs(w));
            e2 = std::max(e2, std::abs(cd(regs[t].v[n1].x, regs[t].v[n1].y) - w));
        }
    printf("R3=%2d L=%4d: n2p err %.3e (rel %.2e), perm bijective: %s, p2n(n2p(x)) err rel %.2e\n", R3, G::L, e1, e1 / xmax,
           bad ? "NO" : "yes", e2 / ymax);
    return (e1 / xmax < 2e-6 && !bad && e2 / ymax < 4e-6) ? 0 : 1;
}

// Largest error of n2p (x -> X, relative to max |X|) and of p2n alone (permuted z -> y[n] = sum_k z[k] W^{nk}, relative
// to max |y|) over `trials` random inputs, with the pass-1 / pass-3 twiddles of thread t from src(t).
template <int R3, class Src>
void source_errors(const std::vector<float2>& tw, Src src, int trials, double& en2p, double& ep2n) {
    using G = Geo<R3>;
    const float2* tw2 = tw.data() + G::TW1;
    std::vector<float2> ea(G::EX), eb(G::EX), x(G::L);
    struct Regs { float2 v[16]; };
    std::vector<Regs> regs(G::T);
    std::vector<cd> W(G::L);
    for (int m = 0; m < G::L; ++m) W[m] = std::polar(1.0, -2.0 * M_PI * m / G::L);
    auto dft = [&](const std::vector<float2>& in, std::vector<cd>& out) {
        out.assign(G::L, 0);
        for (int k = 0; k < G::L; ++k)
            for (int n = 0; n < G::L; ++n) out[k] += cd(in[n].x, in[n].y) * W[(long long)n * k % G::L];
    };
    std::mt19937 rng(4321 + R3);
    std::normal_distribution<float> nd;
    std::vector<cd> X;
    en2p = ep2n = 0;
    for (int trial = 0; trial < trials; ++trial) {
        for (auto& v : x) v = make_float2(nd(rng), nd(rng));
        dft(x, X);
        for (int t = 0; t < G::T; ++t) for (int n1 = 0; n1 < 16; ++n1) regs[t].v[n1] = x[n1 * G::T + t];
        for (int t = 0; t < G::T; ++t) n2p_pass1<R3>(regs[t].v, t, ea.data(), src(t));
        for (int t = 0; t < G::T; ++t) n2p_pass2<R3>(regs[t].v, t, ea.data(), eb.data(), Tw2Table<R3>{tw2});
        for (int t = 0; t < G::T; ++t) n2p_pass3<R3>(regs[t].v, t, eb.data());
        double e = 0, xmax = 0;
        for (auto& v : X) xmax = std::max(xmax, std::abs(v));
        for (int t = 0; t < G::T; ++t)
            for (int r = 0; r < 16; ++r) e = std::max(e, std::abs(cd(regs[t].v[r].x, regs[t].v[r].y) - X[perm_freq<R3>(t, r)]));
        en2p = std::max(en2p, e / xmax);
        // p2n of x laid out in permuted order: register r of thread t holds z[perm_freq(t, r)] = x[perm_freq(t, r)]
        for (int t = 0; t < G::T; ++t) for (int r = 0; r < 16; ++r) regs[t].v[r] = x[perm_freq<R3>(t, r)];
        for (int t = 0; t < G::T; ++t) p2n_pass1<R3>(regs[t].v, t, eb.data());
        for (int t = 0; t < G::T; ++t) p2n_pass2<R3>(regs[t].v, t, eb.data(), ea.data(), Tw2Table<R3>{tw2});
        for (int t = 0; t < G::T; ++t) p2n_pass3<R3>(regs[t].v, t, ea.data(), src(t));
        e = 0;                                   // y = DFT(x): the DFT matrix is symmetric, so X is the wanted output
        for (int t = 0; t < G::T; ++t)
            for (int n1 = 0; n1 < 16; ++n1) e = std::max(e, std::abs(cd(regs[t].v[n1].x, regs[t].v[n1].y) - X[n1 * G::T + t]));
        ep2n = std::max(ep2n, e / xmax);
    }
}

// Tw1Seeds<8> (frame_pass_kernel's pass-1 / pass-3 twiddles) against float64 and, through whole transforms, against
// the table it replaces
int seeds() {
    constexpr int R3 = 8;
    using G = Geo<R3>;
    std::vector<float2> tw;
    make_tw<R3>(tw);
    const float2* tw1 = tw.data();
    double ulp = 0;                              // largest component error of a twiddle, in units of 2^-23 (1 ulp of 1.0)
    for (int t = 0; t < G::T; ++t) {
        const Tw1Seeds<R3> s(tw1, t);
        for (int k1 = 1; k1 < 16; ++k1) {
            const float2 w = s(t, k1);
            const double a = -2.0 * M_PI * (double)((long long)t * k1 % G::L) / G::L;
            ulp = std::max(ulp, std::max(std::abs(w.x - cos(a)), std::abs(w.y - sin(a))) * 8388608.0);
        }
    }
    double tn, tp, sn, sp;
    source_errors<R3>(tw, [&](int) { return Tw1Table<R3>{tw1}; }, 4, tn, tp);
    source_errors<R3>(tw, [&](int t) { return Tw1Seeds<R3>(tw1, t); }, 4, sn, sp);
    printf("twiddle_ulp=%.4f table_n2p=%.4e seeded_n2p=%.4e table_p2n=%.4e seeded_p2n=%.4e smem_seeded_float2=%d "
           "smem_table_float2=%d\n", ulp, tn, sn, tp, sp, SmemSeeded<R3, Tw2Table<R3>>::SMEM_FLOAT2, G::SMEM_FLOAT2);
    return 0;
}

// Shared-memory wavefronts of one warp's access: `addr[l]` is lane l's byte address, each lane reads `bytes` from it.
// The 32 banks are 4 bytes wide; a word read by several lanes is fetched once, and a bank serves one word per
// wavefront, so the count is the largest number of distinct words any bank holds (at least one per 128 bytes).
int wavefronts(const int* addr, int bytes) {
    std::vector<std::vector<int>> bank(32);
    int words = 0;
    for (int l = 0; l < 32; ++l)
        for (int b = 0; b < bytes; b += 4) {
            const int w = (addr[l] + b) / 4;
            auto& v = bank[w % 32];
            if (std::find(v.begin(), v.end(), w) == v.end()) { v.push_back(w); ++words; }
        }
    int n = (words + 31) / 32;
    for (auto& v : bank) n = std::max(n, (int)v.size());
    return n;
}

// Tw2Rows<8> (frame_pass_kernel's pass-2 twiddles): the staged rows against the table, the wavefronts of the pair loads
// of every warp against those of the table's loads, and whole transforms (seeded pass 1 / pass 3, as the kernel runs
// them) with the rows against the same with the table, bit for bit
int rows() {
    constexpr int R3 = 8;
    using G = Geo<R3>;
    using Rows = Tw2Rows<R3>;
    std::vector<float2> tw;
    make_tw<R3>(tw);
    const float2* tw1 = tw.data();
    const float2* tw2 = tw.data() + G::TW1;
    std::vector<float4> buf(Rows::FLOAT2 / 2);                    // 16-byte aligned, as the kernel's shared memory
    float2* rw = reinterpret_cast<float2*>(buf.data());
    for (int i = 0; i < Rows::FLOAT2; ++i) rw[i] = Rows::staged(tw2, i);
    int values_ok = 1;
    for (int n3 = 0; n3 < R3; ++n3)
        for (int k2 = 0; k2 < Rows::STRIDE; ++k2) {
            const float2 got = rw[n3 * Rows::STRIDE + k2];
            const float2 want = k2 < 16 ? tw2[k2 * R3 + n3] : make_float2(0.f, 0.f);
            values_ok &= got.x == want.x && got.y == want.y;
        }
    int loaded_ok = 1;                                           // what load() hands pass 2: w[k2], k2 = 1..15
    for (int n3 = 0; n3 < R3; ++n3) {
        float2 w[16];
        Rows{rw}.load(w, n3);
        for (int k2 = 1; k2 < 16; ++k2) loaded_ok &= w[k2].x == tw2[k2 * R3 + n3].x && w[k2].y == tw2[k2 * R3 + n3].y;
    }
    // lane l of warp q is thread t = 32 q + l, n3 = t mod R3; byte addresses relative to the 16-byte aligned table
    int wf_rows = 0, wf_table = 0, aligned = 1;
    for (int q = 0; q < G::T / 32; ++q) {
        int addr[32];
        for (int h = 0; h < 8; ++h) {                            // pairs (2h, 2h + 1): one 128-bit load each
            for (int l = 0; l < 32; ++l) addr[l] = ((32 * q + l) % R3) * Rows::STRIDE * 8 + 16 * h;
            for (int l = 0; l < 32; ++l) aligned &= addr[l] % 16 == 0;
            wf_rows = std::max(wf_rows, wavefronts(addr, 16));
        }
        for (int k2 = 1; k2 < 16; ++k2) {                        // tw2[k2 R3 + n3]: one 64-bit load each
            for (int l = 0; l < 32; ++l) addr[l] = (k2 * R3 + (32 * q + l) % R3) * 8;
            wf_table = std::max(wf_table, wavefronts(addr, 8));
        }
    }
    // n2p and p2n with the rows against the same with the table
    std::mt19937 rng(2468);
    std::normal_distribution<float> nd;
    std::vector<float2> ea(G::EX), eb(G::EX), x(G::L);
    struct Regs { float2 v[16]; };
    std::vector<Regs> a(G::T), b(G::T);
    int bitwise = 1;
    for (int trial = 0; trial < 4; ++trial) {
        for (auto& v : x) v = make_float2(nd(rng), nd(rng));
        for (int pass = 0; pass < 2; ++pass) {
            std::vector<Regs>& regs = pass ? b : a;
            for (int t = 0; t < G::T; ++t) for (int n1 = 0; n1 < 16; ++n1) regs[t].v[n1] = x[n1 * G::T + t];
            for (int t = 0; t < G::T; ++t) n2p_pass1<R3>(regs[t].v, t, ea.data(), Tw1Seeds<R3>(tw1, t));
            for (int t = 0; t < G::T; ++t)
                if (pass) n2p_pass2<R3>(regs[t].v, t, ea.data(), eb.data(), Rows{rw});
                else n2p_pass2<R3>(regs[t].v, t, ea.data(), eb.data(), Tw2Table<R3>{tw2});
            for (int t = 0; t < G::T; ++t) n2p_pass3<R3>(regs[t].v, t, eb.data());
            for (int t = 0; t < G::T; ++t) p2n_pass1<R3>(regs[t].v, t, eb.data());
            for (int t = 0; t < G::T; ++t)
                if (pass) p2n_pass2<R3>(regs[t].v, t, eb.data(), ea.data(), Rows{rw});
                else p2n_pass2<R3>(regs[t].v, t, eb.data(), ea.data(), Tw2Table<R3>{tw2});
            for (int t = 0; t < G::T; ++t) p2n_pass3<R3>(regs[t].v, t, ea.data(), Tw1Seeds<R3>(tw1, t));
        }
        for (int t = 0; t < G::T; ++t)
            for (int r = 0; r < 16; ++r) bitwise &= a[t].v[r].x == b[t].v[r].x && a[t].v[r].y == b[t].v[r].y;
    }
    printf("rows_values_ok=%d rows_loaded_ok=%d rows_aligned=%d rows_wavefronts=%d table_wavefronts=%d "
           "rows_bit_identical=%d smem_rows_float2=%d smem_seeded_float2=%d\n", values_ok, loaded_ok, aligned, wf_rows,
           wf_table, bitwise, SmemSeeded<R3, Rows>::SMEM_FLOAT2, SmemSeeded<R3, Tw2Table<R3>>::SMEM_FLOAT2);
    return 0;
}

int main(int argc, char** argv) {
    if (argc > 1 && std::string(argv[1]) == "seeds") return seeds();
    if (argc > 1 && std::string(argv[1]) == "rows") return rows();
    int rc = run<4>() | run<8>() | run<16>();
    printf(rc ? "FAIL\n" : "OK\n");
    return rc;
}
