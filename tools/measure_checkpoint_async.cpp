// Node-drive harness of tools/measure_checkpoint_async.py: drives dsm::SurfelMapNode through measure_node.cpp's message
// script as a node does, without synchronising per frame, and checkpoints every `every` frames.
// Usage: measure_checkpoint_async W H fx fy cx cy far near drift_free_poses frames.bin script.bin mode every dir
//   frames.bin, script.bin: as measure_node.cpp (the publish field is ignored)
//   mode 0: no checkpoint.
//   mode 1: save_state_async when `every` frames have passed since the last save, polled with wait_state_saved(false)
//           before each frame's callbacks; a save that falls due while the previous one is still written is skipped
//           (the policy of INTEGRATION.md section 4: the node never waits).
//   mode 2: the blocking save_state every `every` frames.
//   mode 3: save_state_async every `every` frames, waiting (wait_state_saved(true)) for a previous one still in flight.
// Prints one JSON object: the wall time of the whole drive (one synchronisation at its end), per frame, the checkpoints
// written, the frames on which a due save was put off because the previous one was still written (mode 1) and the
// host time spent in blocking waits (mode 3), and the host time inside the save calls themselves.
#include <string>
#include "measure_drive.hpp"

int main(int argc, char **argv)
{
    if (argc != 15) return 2;
    const int W = atoi(argv[1]), mode = atoi(argv[12]), every = atoi(argv[13]);
    const std::string dir = argv[14];
    if (every < 1) return 5;
    Drive d;
    if (!d.load(argv)) return 5;
    const int T = (int)d.msgs.size();
    DriveNode node(argv);
    if (const int e = node.setup_code()) return e;
    if ((mode == 1 || mode == 3) && node.enable_checkpoints() != DSM_OK) return 6;
    int saves = 0, skipped = 0, in_flight = 0, since = 0;
    double wait_ms = 0, call_ms = 0;
    const clk::time_point t0 = clk::now();
    for (int t = 0; t < T; t++)
    {
        const DriveMsg &m = d.msgs[(size_t)t];
        if (in_flight)
        { // the poll of the next call
            bool fin = false;
            if (node.wait_state_saved(false, &fin) != DSM_OK) return 6;
            in_flight = !fin;
        }
        int rc = m.orb(node);
        if (rc == DSM_OK) rc = d.images(node, m, W);
        if (rc != DSM_OK) return 6;
        if (mode != 0 && ++since >= every)
        {
            const std::string p = dir + "/node" + std::to_string(saves % 2) + ".dsm";
            if (mode == 1 && in_flight)
            {
                skipped++; // still due on the next frame
                continue;
            }
            if (mode == 3 && in_flight)
            {
                const clk::time_point w = clk::now();
                if (node.wait_state_saved(true, nullptr) != DSM_OK) return 6;
                wait_ms += ms(w, clk::now());
            }
            const clk::time_point c = clk::now();
            rc = mode == 2 ? node.save_state(p) : node.save_state_async(p);
            call_ms += ms(c, clk::now());
            in_flight = mode != 2;
            if (rc != DSM_OK) return 6;
            saves++;
            since = 0;
        }
    }
    dsm_sync(node.context());
    const double total = ms(t0, clk::now());
    // the last checkpoint's write finishes outside the timed drive, as it would behind the node's next frames
    if (in_flight && node.wait_state_saved(true, nullptr) != DSM_OK) return 6;
    int n_store = 0;
    if (dsm_inactive_size(node.context(), &n_store, nullptr) != DSM_OK) return 6;
    std::printf("{\"frames\": %d, \"total_ms\": %.3f, \"ms_per_frame\": %.4f, \"saves\": %d, \"skipped\": %d, \"wait_ms\": %.3f, "
                "\"save_call_ms\": %.3f, \"store_surfels\": %d}\n",
                T, total, total / (T ? T : 1), saves, skipped, wait_ms, call_ms, n_store);
    return 0;
}
