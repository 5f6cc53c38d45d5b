package ch.sqooba.kao;

/**
 * JNI view of include/kao.h.  One call replaces "write the LP (README.md:139-185), run lp_solve
 * (README.md:135-136), parse the variables".  UNCOMPILED in this repository (no JDK in the image).
 */
public final class KaoNative {
    static { System.loadLibrary("kaojni"); }

    private KaoNative() {}

    /** kao_options.flags: kao_result objective bound from the flow relaxations (host) */
    public static final int FLAG_BOUND = 0x400;
    /** kao_options.flags: also the Lagrangian LP bound on the GPU (docs/MODEL.md 9): proves optima the flow bound cannot */
    public static final int FLAG_LP_BOUND = 0x1000;

    /** kao_version() */
    public static native int version();

    /**
     * kao_solve().  Tables are row-major over dense broker indices 0..B-1 (position in the sorted
     * target broker list, README.md:48).
     *
     * @param rackOf  [B]    rack index per broker (README.md:27-29)
     * @param wF      [P*B]  follower weights (README.md:145-146), unsigned 16-bit values in shorts
     * @param wL      [P*B]  leader weights (README.md:131-133)
     * @param bounds  [4*B + 2*R + 2] rep_lo, rep_hi, ldr_lo, ldr_hi (each [B]), rack_lo, rack_hi
     *                (each [R]), ppr_lo, ppr_hi — C3, C4, C6, C7 right-hand sides (README.md:158-180)
     * @param cur     [P*RFcur] current assignment, leader first, -1 = absent (README.md:52-63)
     * @param replicasOut [P*RF] result, leader first (README.md:67-78, :88)
     * @param nGpus   1, or N: every round is sharded over N GPUs of this process (device .. device+N-1)
     * @param flags   kao_options.flags: restarts | KAO_FLAG_DELTA (0x100) | KAO_FLAG_SPREAD_RESTARTS (0x800) | FLAG_BOUND | FLAG_LP_BOUND | KAO_FLAG_PATIENCE(n) (n << 16)
     * @param statsOut [8] objective, violation, replica moves, candidates evaluated, objective upper
     *                bound, proven optimal (0/1), rounds run, GPUs used
     * @return 0 ok, 1 no feasible assignment found; throws KaoException on argument/CUDA errors
     */
    public static native int solve(int P, int B, int R, int RF, int RFcur, byte[] rackOf, short[] wF,
                                   short[] wL, int[] bounds, int[] cur, long seed, int rounds,
                                   int roundSize, int device, int nGpus, int flags, int[] replicasOut,
                                   long[] statsOut);

    public static final class KaoException extends RuntimeException {
        public final int code;
        public KaoException(int code, String message) { super(message); this.code = code; }
    }
}
