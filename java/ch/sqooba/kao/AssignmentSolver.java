package ch.sqooba.kao;

import java.io.IOException;
import java.nio.charset.StandardCharsets;
import java.nio.file.Files;
import java.nio.file.Paths;
import java.util.*;

/**
 * The tool's command line on top of KaoNative.solve — the place where the reference builds its LP
 * (README.md:139-185) and shells to lp_solve (README.md:135-136).  Same flags, defaults and output as
 * kao-cli (kafka_assignment_optimizer_b200/csrc/kao_cli.cpp), same model defaults as docs/MODEL.md §1.
 * UNCOMPILED in this repository (no JDK in the image).
 *
 * <pre>
 * java -Djava.library.path=. ch.sqooba.kao.AssignmentSolver --assignment current.json \
 *      --brokers 0,1,2,...,18 --racks 0:a,1:b,... [--rf 2] [--rounds 256] [--round-size 32768]
 *      [--restarts 1] [--seed 24301] [--device 0] [--gpus 1] [--spread-restarts] [--delta] [--patience N] [--certificate] [--lp-certificate] [--stats]
 * </pre>
 * in:  the JSON `kafka-reassign-partitions --generate` prints (README.md:52-63), the target broker list
 *      (README.md:48), broker:rack pairs (README.md:27-29);
 * out: the JSON `kafka-reassign-partitions --reassignment-json-file` takes (README.md:67-78), leader first.
 */
public final class AssignmentSolver {
    private static final int FLAG_DELTA = 0x100;
    private static final int FLAG_BOUND = 0x400;             // flow-bound certificate: the result can say "proven optimal"
    private static final int FLAG_SPREAD_RESTARTS = 0x800;   // --gpus N: the restarts side by side, one per GPU at a time

    /** One row of the assignment JSON. */
    static final class Row {
        String topic;
        int partition;
        int[] replicas;
    }

    /** current[p] = broker ids, leader first (README.md:52-63); brokers = target list (README.md:48). */
    public static int[][] solve(int[][] current, int[] brokers, Map<Integer, String> rackOfBroker, int rf,
                                long seed, int rounds, int roundSize, int device, int nGpus, int flags, long[] stats) {
        int[] ids = Arrays.stream(brokers).sorted().distinct().toArray();
        int P = current.length, B = ids.length;
        Map<Integer, Integer> dense = new HashMap<>();
        for (int i = 0; i < B; i++) dense.put(ids[i], i);
        List<String> racks = new ArrayList<>(new TreeSet<>(rackOfBroker.values()));
        racks.removeIf(r -> Arrays.stream(ids).noneMatch(b -> rackOfBroker.get(b).equals(r)));
        int R = racks.size();
        byte[] rackOf = new byte[B];
        long[] size = new long[R];
        for (int i = 0; i < B; i++) { rackOf[i] = (byte) racks.indexOf(rackOfBroker.get(ids[i])); size[rackOf[i]]++; }
        int rfCur = Math.max(1, Arrays.stream(current).mapToInt(c -> c.length).max().orElse(1));
        int[] cur = new int[P * rfCur];
        Arrays.fill(cur, -1);
        short[] wF = new short[P * B], wL = new short[P * B];
        int[] WL = {4, 2, 1}, WF = {2, 2, 1};                       // README.md:146, :131-133
        for (int p = 0; p < P; p++)
            for (int i = 0; i < current[p].length; i++) {
                Integer d = dense.get(current[p][i]);
                if (d == null) continue;                           // broker leaves the cluster
                cur[p * rfCur + i] = d;
                wF[p * B + d] = (short) (i < 3 ? WF[i] : 1);
                wL[p * B + d] = (short) (i < 3 ? WL[i] : 1);
            }
        long tot = (long) P * rf;
        int[] bounds = new int[4 * B + 2 * R + 2];
        for (int b = 0; b < B; b++) {
            bounds[b] = (int) (tot / B);         bounds[B + b] = (int) ((tot + B - 1) / B);       // C3
            bounds[2 * B + b] = P / B;           bounds[3 * B + b] = (P + B - 1) / B;             // C4
        }
        for (int r = 0; r < R; r++) {                                                           // C6
            bounds[4 * B + r] = (int) (tot * size[r] / B);
            bounds[4 * B + R + r] = (int) ((tot * size[r] + B - 1) / B);
        }
        bounds[4 * B + 2 * R] = rf / R;  bounds[4 * B + 2 * R + 1] = (rf + R - 1) / R;            // C7
        int[] out = new int[P * rf];
        KaoNative.solve(P, B, R, rf, rfCur, rackOf, wF, wL, bounds, cur, seed, rounds, roundSize, device, nGpus, flags,
                        out, stats);
        int[][] res = new int[P][];
        for (int p = 0; p < P; p++) {
            int n = 0;
            for (int i = 0; i < rf; i++) if (out[p * rf + i] >= 0) n++;
            res[p] = new int[n];
            for (int i = 0, k = 0; i < rf; i++) if (out[p * rf + i] >= 0) res[p][k++] = ids[out[p * rf + i]];
        }
        return res;                                                // leader first (README.md:67-78, :88)
    }

    // ---- the two JSON shapes of README.md:52-63 / :67-78; nothing else is ever parsed or printed here
    /** {"version":1,"partitions":[{"topic":"t","partition":0,"replicas":[7,18]}, ...]} */
    static List<Row> parseAssignment(String text) {
        List<Row> rows = new ArrayList<>();
        int at = text.indexOf("\"partitions\"");
        if (at < 0) throw new IllegalArgumentException("no \"partitions\" array in the assignment JSON");
        int i = text.indexOf('[', at);
        while (true) {
            int open = text.indexOf('{', i), close = text.indexOf(']', i);
            if (open < 0 || (close >= 0 && close < open)) break;            // end of the partitions array
            int end = text.indexOf('}', open);
            String obj = text.substring(open + 1, end);
            Row r = new Row();
            r.topic = stringField(obj, "topic");
            r.partition = Integer.parseInt(scalarField(obj, "partition"));
            int lb = obj.indexOf('[', obj.indexOf("\"replicas\"")), rb = obj.indexOf(']', lb);
            String list = obj.substring(lb + 1, rb).trim();
            r.replicas = list.isEmpty() ? new int[0]
                    : Arrays.stream(list.split(",")).mapToInt(s -> Integer.parseInt(s.trim())).toArray();
            rows.add(r);
            i = end + 1;
        }
        if (rows.isEmpty()) throw new IllegalArgumentException("no partitions in the assignment");
        return rows;
    }

    private static String scalarField(String obj, String name) {
        int k = obj.indexOf("\"" + name + "\"");
        if (k < 0) throw new IllegalArgumentException("missing field " + name);
        int c = obj.indexOf(':', k) + 1, e = c;
        while (e < obj.length() && obj.charAt(e) != ',' && obj.charAt(e) != '}') e++;
        return obj.substring(c, e).trim();
    }

    private static String stringField(String obj, String name) {
        String v = scalarField(obj, name);
        if (v.length() < 2 || v.charAt(0) != '"') throw new IllegalArgumentException("field " + name + " is not a string");
        return v.substring(1, v.lastIndexOf('"'));
    }

    static String reassignmentJson(List<Row> rows, int[][] replicas) {
        StringBuilder sb = new StringBuilder("{\"version\":1,\"partitions\":[\n");
        for (int p = 0; p < rows.size(); p++) {
            sb.append("    {\"topic\":\"").append(rows.get(p).topic).append("\",\"partition\":").append(rows.get(p).partition)
              .append(",\"replicas\":[");
            for (int i = 0; i < replicas[p].length; i++) sb.append(i == 0 ? "" : ",").append(replicas[p][i]);
            sb.append("]}").append(p + 1 < rows.size() ? "," : "").append('\n');
        }
        return sb.append("]}\n").toString();
    }

    private static int usage() {
        System.err.println("usage: AssignmentSolver --assignment FILE|- --brokers 0,1,2 --racks 0:a,1:b,2:a [--rf N]\n"
                + "       [--rounds 256] [--round-size 32768] [--restarts 1] [--seed 24301] [--device 0] [--gpus 1]"
                + " [--spread-restarts] [--delta] [--patience N] [--certificate] [--lp-certificate] [--stats]");
        return 2;
    }

    /** Exit status as kao-cli: 0 ok, 1 error, 2 usage, 3 no assignment satisfying every constraint was found. */
    public static void main(String[] argv) throws IOException {
        Map<String, String> a = new HashMap<>();
        boolean stats = false, delta = false, spread = false, certificate = false, lpCertificate = false;
        for (int i = 0; i < argv.length; i++) {
            String k = argv[i];
            if (k.equals("--stats")) { stats = true; continue; }
            if (k.equals("--delta")) { delta = true; continue; }
            if (k.equals("--spread-restarts")) { spread = true; continue; }
            if (k.equals("--certificate")) { certificate = true; continue; }
            if (k.equals("--lp-certificate")) { lpCertificate = true; continue; }   // Lagrangian LP bound on the GPU
            if (!k.startsWith("--") || i + 1 >= argv.length) System.exit(usage());
            a.put(k.substring(2), argv[++i]);
        }
        if (!a.containsKey("assignment") || !a.containsKey("brokers") || !a.containsKey("racks")) System.exit(usage());
        try {
            String path = a.get("assignment");
            String text = path.equals("-") ? new String(System.in.readAllBytes(), StandardCharsets.UTF_8)
                    : new String(Files.readAllBytes(Paths.get(path)), StandardCharsets.UTF_8);
            List<Row> rows = parseAssignment(text);
            int[] brokers = Arrays.stream(a.get("brokers").split(",")).mapToInt(s -> Integer.parseInt(s.trim())).toArray();
            Map<Integer, String> racks = new HashMap<>();
            for (String t : a.get("racks").split(",")) {
                int c = t.indexOf(':');
                if (c < 0) throw new IllegalArgumentException("rack map entries look like id:rack");
                racks.put(Integer.parseInt(t.substring(0, c).trim()), t.substring(c + 1));
            }
            int rf = rows.stream().mapToInt(r -> r.replicas.length).max().orElse(1);
            if (a.containsKey("rf")) rf = Integer.parseInt(a.get("rf"));
            int[][] current = rows.stream().map(r -> r.replicas).toArray(int[][]::new);
            int flags = Math.min(255, Math.max(1, Integer.parseInt(a.getOrDefault("restarts", "1"))));
            if (delta) flags |= FLAG_DELTA;
            if (spread) flags |= FLAG_SPREAD_RESTARTS;
            if (certificate) flags |= FLAG_BOUND;
            if (lpCertificate) flags |= KaoNative.FLAG_LP_BOUND;
            if (a.containsKey("patience")) flags |= Math.min(65535, Math.max(0, Integer.parseInt(a.get("patience")))) << 16;
            long[] st = new long[8];
            int[][] res = solve(current, brokers, racks, rf, Long.decode(a.getOrDefault("seed", "24301")),
                                Integer.parseInt(a.getOrDefault("rounds", "256")),
                                Integer.parseInt(a.getOrDefault("round-size", "32768")),
                                Integer.parseInt(a.getOrDefault("device", "0")),
                                Integer.parseInt(a.getOrDefault("gpus", "1")), flags, st);
            System.out.print(reassignmentJson(rows, res));
            if (stats)
                System.err.printf("objective %d (upper bound %d%s), violation %d, replica moves %d, %d candidates, %d GPU(s)%n",
                                  st[0], st[4], st[5] != 0 ? ": proven optimal" : "", st[1], st[2], st[3], st[7]);
            if (st[1] != 0) {
                System.err.println("warning: no assignment satisfying every constraint was found (violation " + st[1] + ")");
                System.exit(3);
            }
        } catch (KaoNative.KaoException | IllegalArgumentException e) {
            System.err.println("AssignmentSolver: " + e.getMessage());
            System.exit(1);
        }
    }
}
