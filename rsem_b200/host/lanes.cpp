// Devices, and the lanes of the batch executables: contexts opened side by side, the manifest lines handed out in order.
#include <algorithm>
#include <cstdlib>
#include <sstream>
#include <thread>

#include "host.hpp"

namespace host {

std::vector<int> gpu_devices() {
    std::vector<int> devices;
    if (const char* e = getenv("RSEM_B200_DEVICES")) {  // e.g. "0,1,2,3"
        for (const char* q = e; *q;) {
            devices.push_back(atoi(q));
            while (*q && *q != ',') ++q;
            if (*q == ',') ++q;
        }
    }
    if (devices.size() <= 1) {
        const char* one = getenv("RSEM_B200_DEVICE");
        devices.assign(1, one ? atoi(one) : devices.empty() ? 0 : devices[0]);
    }
    return devices;
}

namespace {

LaneContexts open_contexts(const std::vector<int>& devices, bool want_free) {
    const size_t n = devices.size();
    LaneContexts out;
    out.ctx.assign(n, nullptr);
    out.free.assign(n, 0);
    const char* e = getenv("RSEM_B200_BATCH_ARENA_BYTES");
    const uint64_t set = e ? strtoull(e, nullptr, 10) : 0;   // 0 is the default, as unset
    out.arena.assign(n, set);
    const bool share = n > 1 && set == 0;
    std::vector<std::string> err(n);
    std::vector<int> distinct;
    for (int d : devices)
        if (std::find(distinct.begin(), distinct.end(), d) == distinct.end()) distinct.push_back(d);
    // per device: its free memory, then the contexts of its lanes; the devices side by side
    auto open_device = [&](int d) {
        std::vector<size_t> mine;
        for (size_t k = 0; k < n; ++k)
            if (devices[k] == d) mine.push_back(k);
        const std::string where = n > 1 ? "device " + std::to_string(d) + ": " : "";
        if (share || want_free) {
            uint64_t free_b = 0;
            if (rsem_b200_device_free_bytes(d, &free_b) != 0) {
                err[mine[0]] = "rsem_b200: " + where + "device_free_bytes failed: " + rsem_b200_last_error();
                return;
            }
            for (size_t k : mine) {
                out.free[k] = free_b;
                if (share) out.arena[k] = free_b / 2 / mine.size();
            }
        }
        for (size_t k : mine)
            if (rsem_b200_ctx_create(d, &out.ctx[k]) != 0) {
                err[k] = "rsem_b200: " + where + "ctx_create failed: " + rsem_b200_last_error();
                return;
            }
    };
    {
        std::vector<std::thread> pool;
        for (size_t j = 1; j < distinct.size(); ++j) pool.emplace_back(open_device, distinct[j]);
        open_device(distinct[0]);
        for (auto& th : pool) th.join();
    }
    for (const std::string& m : err)
        if (!m.empty()) {
            out.err = m;
            break;
        }
    return out;
}

}  // namespace

LaneContexts open_lanes(const std::vector<int>& devices) { return open_contexts(devices, false); }

LaneContexts open_lanes_measured(const std::vector<int>& devices) { return open_contexts(devices, true); }

size_t Claims::next() {
    if (failed_) return n_;
    return std::min(n_, i_.fetch_add(1));
}

void Claims::fail(const std::string& msg) {
    std::lock_guard<std::mutex> g(mu_);
    if (failed_) return;
    msg_ = msg;
    failed_ = true;
}

bool Claims::failed() { return failed_; }

std::string Claims::message() {
    std::lock_guard<std::mutex> g(mu_);
    return msg_;
}

std::vector<ManifestLine> manifest_lines(const std::string& path) {
    std::vector<char> buf = slurp(path);
    std::istringstream in(std::string(buf.begin(), buf.end()));
    std::vector<ManifestLine> lines;
    std::string raw;
    for (int no = 1; std::getline(in, raw); ++no) {
        std::istringstream ls(raw);
        ManifestLine l{no, {}};
        for (std::string w; ls >> w;) l.f.push_back(w);
        if (!l.f.empty()) lines.push_back(std::move(l));
    }
    return lines;
}

void refuse(const std::string& manifest, int no, const std::string& why) {
    die(manifest + " line " + std::to_string(no) + ": " + why);
}

std::string sample_at(const std::string& name, const std::string& manifest, int no) {
    return "sample " + name + " (" + manifest + " line " + std::to_string(no) + ")";
}

}  // namespace host
