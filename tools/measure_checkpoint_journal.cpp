// Node-drive harness of tools/measure_checkpoint_journal.py: drives dsm::SurfelMapNode through measure_node.cpp's message
// script as a node does, without synchronising per frame, and checkpoints once `every` frames have passed, skipping a
// due save while the previous one is still written (the policy of INTEGRATION.md section 4).
// Usage: measure_checkpoint_journal W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode every dir
//   frames.bin, script.bin: as measure_node.cpp (the publish field is ignored)
//   mode 0: no checkpoint.  mode 1: save_state_async (a whole file each time).  mode 2: save_state_incremental.
// Prints one JSON object: the wall time of the drive (one synchronisation at its end) per frame, the saves, the saves
// put off, and for every finished save the bytes it wrote (the file for a whole file or a base, the record otherwise)
// and whether it was a base.
#include <sys/stat.h>

#include <string>
#include "measure_drive.hpp"

static long long size_of(const std::string &p)
{
    struct stat st;
    return stat(p.c_str(), &st) == 0 ? (long long)st.st_size : -1;
}

int main(int argc, char **argv)
{
    if (argc != 15) return 2;
    const int W = atoi(argv[1]), mode = atoi(argv[12]), every = atoi(argv[13]);
    const std::string dir = argv[14], path = dir + "/node_journal.dsm";
    if (every < 1) return 5;
    Drive d;
    if (!d.load(argv)) return 5;
    const int T = (int)d.msgs.size();
    DriveNode node(argv);
    if (const int e = node.setup_code()) return e;
    if (mode != 0 && node.enable_checkpoints() != DSM_OK) return 6;
    int saves = 0, skipped = 0, in_flight = 0, since = 0;
    long long journal = 0;
    std::vector<long long> bytes;
    std::vector<int> base;
    auto finished = [&]() { // the save just retired: what it wrote
        const long long j = size_of(path + ".journal");
        const bool b = mode == 1 || j < journal || j == 32;
        bytes.push_back(b ? size_of(path) : j - journal);
        base.push_back(b ? 1 : 0);
        journal = j;
    };
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T; t++)
    {
        const DriveMsg &m = d.msgs[(size_t)t];
        if (in_flight)
        { // the poll of the next call
            bool fin = false;
            if (node.wait_state_saved(false, &fin) != DSM_OK) return 6;
            in_flight = !fin;
            if (fin) finished();
        }
        int rc = m.orb(node);
        if (rc == DSM_OK) rc = d.images(node, m, W);
        if (rc != DSM_OK) return 6;
        if (mode != 0 && ++since >= every)
        {
            if (in_flight)
            {
                skipped++; // still due on the next frame
                continue;
            }
            rc = mode == 1 ? node.save_state_async(path) : node.save_state_incremental(path);
            if (rc != DSM_OK) return 6;
            in_flight = 1;
            saves++;
            since = 0;
        }
    }
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    if (in_flight)
    {
        if (node.wait_state_saved(true, nullptr) != DSM_OK) return 6;
        finished();
    }
    std::printf("{\"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"saves\": %d, \"skipped\": %d, \"bytes\": [", T, total,
                total / (T ? T : 1), saves, skipped);
    for (size_t i = 0; i < bytes.size(); i++) std::printf("%s%lld", i ? ", " : "", bytes[i]);
    std::printf("], \"base\": [");
    for (size_t i = 0; i < base.size(); i++) std::printf("%s%d", i ? ", " : "", base[i]);
    std::printf("]}\n");
    return 0;
}
