// circom_cuda_prover <circuit.r1cs> <circuit.zkey> <witness.wtns | dir> <proof.json> <public.json>
//
// rapidsnark's `prover <circuit.zkey> <witness.wtns> <proof.json> <public.json>` plus the .r1cs: this library's quotient
// reads A and B from the R1CS (the .zkey's coefficient section is only checked against it).  A directory of witnesses
// (its *.wtns files, in name order) is proved as one batch on the GPU; proof i and its public signals go to
// <proof>.<i>.json and <public>.<i>.json, and one line per witness names the file it came from.  The blinding is drawn
// by the library (getrandom(2)); `--rs <file>` takes it from a file instead, one line "r s" (decimal) per witness in
// the order above - for reproducing a proof: zero knowledge needs the default draw.  A witness that does not satisfy the
// R1CS is refused before anything is proved.
// A client of the C ABI; device memory comes from the CUDA runtime.
#include <cuda_runtime.h>
#include <dirent.h>
#include <sys/stat.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/circom_b200.h"

namespace {

int die(const std::string &msg) {
    fprintf(stderr, "circom_cuda_prover: %s\n", msg.c_str());
    return 1;
}

std::string lib_error(int rc) { return "error " + std::to_string(rc) + ": " + cw_last_error(); }

bool read_file(const std::string &path, std::string &out) {
    std::ifstream f(path, std::ios::binary);
    if (!f) return false;
    std::stringstream ss;
    ss << f.rdbuf();
    out = ss.str();
    return true;
}

bool write_file(const std::string &path, const std::string &text) {
    FILE *f = fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = fwrite(text.data(), 1, text.size(), f) == text.size();
    return fclose(f) == 0 && ok;
}

// <stem>.<i>.json for <stem>.json (anything else: <path>.<i>)
std::string numbered(const std::string &path, size_t i) {
    const std::string ext = ".json";
    if (path.size() > ext.size() && path.compare(path.size() - ext.size(), ext.size(), ext) == 0)
        return path.substr(0, path.size() - ext.size()) + "." + std::to_string(i) + ext;
    return path + "." + std::to_string(i);
}

// json text through a cw_*_json call: ask for the length, then write
template <class F>
int json_text(F call, std::string &out) {
    size_t len = 0;
    int rc = call(nullptr, 0, &len);
    if (rc) return rc;
    std::vector<char> buf(len + 1);
    if ((rc = call(buf.data(), buf.size(), &len))) return rc;
    out.assign(buf.data(), len);
    return 0;
}

// a decimal below 2^256 into 4 little-endian u64 limbs
bool parse_dec(const std::string &t, uint64_t out[4]) {
    memset(out, 0, 32);
    if (t.empty()) return false;
    for (char ch : t) {
        if (ch < '0' || ch > '9') return false;
        unsigned __int128 carry = (unsigned)(ch - '0');
        for (int i = 0; i < 4; ++i) {
            const unsigned __int128 v = (unsigned __int128)out[i] * 10u + carry;
            out[i] = (uint64_t)v;
            carry = v >> 64;
        }
        if (carry) return false;
    }
    return true;
}

struct Dev {   // one cudaMalloc, freed at scope exit
    void *p = nullptr;
    ~Dev() { if (p) cudaFree(p); }
};

}  // namespace

int main(int argc, char **argv) {
    if (argc != 6 && !(argc == 8 && std::string(argv[6]) == "--rs")) {
        fprintf(stderr, "usage: %s <circuit.r1cs> <circuit.zkey> <witness.wtns | dir> <proof.json> <public.json> [--rs <file>]\n",
                argv[0]);
        return 2;
    }
    const std::string r1cs_path = argv[1], zkey_path = argv[2], wit_path = argv[3], proof_path = argv[4], pub_path = argv[5];
    cw_r1cs *r = nullptr;
    int rc = cw_r1cs_load(r1cs_path.c_str(), &r);
    if (rc) return die(r1cs_path + ": " + lib_error(rc));
    std::string zkey;
    if (!read_file(zkey_path, zkey)) return die("cannot read " + zkey_path);
    cw_groth16_key *k = nullptr;
    if ((rc = cw_groth16_key_create(zkey.data(), zkey.size(), r, 0, &k))) return die(zkey_path + ": " + lib_error(rc));
    zkey.clear();
    zkey.shrink_to_fit();
    uint64_t info[4];
    cw_groth16_key_info(k, info);
    const uint64_t n_vars = info[0], n_public = info[1];

    // the witnesses: one file, or the *.wtns files of a directory in name order
    std::vector<std::string> files;
    struct stat st;
    const bool is_dir = stat(wit_path.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
    if (is_dir) {
        DIR *d = opendir(wit_path.c_str());
        if (!d) return die("cannot open " + wit_path);
        while (dirent *e = readdir(d)) {
            const std::string n = e->d_name;
            if (n.size() > 5 && n.compare(n.size() - 5, 5, ".wtns") == 0) files.push_back(wit_path + "/" + n);
        }
        closedir(d);
        std::sort(files.begin(), files.end());
        if (files.empty()) return die("no .wtns files in " + wit_path);
    } else {
        files.push_back(wit_path);
    }
    const size_t count = files.size();
    std::vector<uint64_t> rows(count * n_vars * 4);
    for (size_t i = 0; i < count; ++i) {
        int prime = -1;
        uint64_t n = 0;
        if ((rc = cw_wtns_read(files[i].c_str(), &prime, &n, nullptr, 0))) return die(files[i] + ": " + lib_error(rc));
        if (prime != CW_PRIME_BN128 || n != n_vars)
            return die(files[i] + ": a bn128 witness of " + std::to_string(n_vars) + " entries is expected, the file has " +
                       std::to_string(n));
        if ((rc = cw_wtns_read(files[i].c_str(), &prime, &n, rows.data() + i * n_vars * 4, n_vars)))
            return die(files[i] + ": " + lib_error(rc));
    }

    std::vector<uint64_t> rs;   // [count][2][4], empty: drawn by the library
    if (argc == 8) {
        std::ifstream f(argv[7]);
        if (!f) return die(std::string("cannot read ") + argv[7]);
        rs.resize(count * 8);
        for (size_t i = 0; i < 2 * count; ++i) {
            std::string t;
            if (!(f >> t) || !parse_dec(t, rs.data() + 4 * i)) return die(std::string(argv[7]) + ": expected 2 decimals per witness");
        }
    }

    // proofs in chunks whose scratch fits half the free device memory
    if (cudaSetDevice(0) != cudaSuccess) return die("no CUDA device");
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    uint32_t chunk = (uint32_t)count;
    uint64_t scratch_b = 0;
    for (;;) {
        if ((rc = cw_groth16_scratch_bytes(k, chunk, &scratch_b))) return die(lib_error(rc));
        if (chunk == 1 || scratch_b <= free_b / 2) break;
        chunk = (chunk + 1) / 2;
    }
    Dev scratch, w_d, p_d;
    if (cudaMalloc(&scratch.p, scratch_b) != cudaSuccess || cudaMalloc(&w_d.p, (size_t)chunk * n_vars * 32) != cudaSuccess ||
        cudaMalloc(&p_d.p, (size_t)chunk * 256) != cudaSuccess)
        return die("out of device memory");
    std::vector<uint64_t> proofs(count * 32);
    for (size_t i0 = 0; i0 < count; i0 += chunk) {
        const uint32_t cn = (uint32_t)std::min<size_t>(chunk, count - i0);
        if (cudaMemcpy(w_d.p, rows.data() + i0 * n_vars * 4, (size_t)cn * n_vars * 32, cudaMemcpyHostToDevice) != cudaSuccess)
            return die("copy to the device failed");
        int64_t bad = -1;
        std::vector<int64_t> first_bad(cn);
        if ((rc = cw_r1cs_check_strided(r, (const uint64_t *)w_d.p, n_vars, 1, cn, 0, first_bad.data(), nullptr)))
            return die(lib_error(rc));
        for (uint32_t i = 0; i < cn; ++i)
            if ((bad = first_bad[i]) >= 0)
                return die(files[i0 + i] + ": the witness violates constraint " + std::to_string(bad));
        if ((rc = cw_groth16_prove_strided(k, r, (const uint64_t *)w_d.p, n_vars, cn, rs.empty() ? nullptr : rs.data() + i0 * 8, (uint64_t *)p_d.p, scratch.p)))
            return die(lib_error(rc));
        if (cudaMemcpy(proofs.data() + i0 * 32, p_d.p, (size_t)cn * 256, cudaMemcpyDeviceToHost) != cudaSuccess)
            return die("copy from the device failed");
    }
    for (size_t i = 0; i < count; ++i) {
        std::string pj, uj;
        const uint64_t *pf = proofs.data() + 32 * i;
        const uint64_t *pub = rows.data() + i * n_vars * 4 + 4;   // w_1 .. w_nPublic
        if ((rc = json_text([&](char *o, size_t c, size_t *l) { return cw_groth16_proof_json(pf, o, c, l); }, pj)) ||
            (rc = json_text([&](char *o, size_t c, size_t *l) { return cw_groth16_public_json(pub, (uint32_t)n_public, o, c, l); }, uj)))
            return die(lib_error(rc));
        const std::string pp = is_dir ? numbered(proof_path, i) : proof_path, up = is_dir ? numbered(pub_path, i) : pub_path;
        if (!write_file(pp, pj) || !write_file(up, uj)) return die("cannot write " + pp + " / " + up);
        if (is_dir) printf("%s -> %s %s\n", files[i].c_str(), pp.c_str(), up.c_str());
    }
    cw_groth16_key_destroy(k);
    cw_r1cs_destroy(r);
    return 0;
}
